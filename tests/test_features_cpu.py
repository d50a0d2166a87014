"""CPU checks of the MFSC feature path: the NumPy reference against first principles (rfft, the mel scale, the filter
shapes, frame counting, the streaming LocalNorm), and the C ABI's argument checks (no kernel is launched)."""
import ctypes

import numpy as np
import pytest

import features_reference as R

FS = 16000


def test_folded_basis_equals_rfft_of_preemphasised_windowed_frame():
    rng = np.random.default_rng(0)
    for frame_ms in (25, 30):
        p = R.Params(FS, frame_ms, 10, 80)
        frames = rng.normal(0, 1000, (7, p.frame))
        direct = np.abs(np.fft.rfft(R.preemphasis(frames) * R.hamming(p.frame)[None, :], n=p.nfft))
        np.testing.assert_allclose(R.magnitude(p, frames), direct, rtol=1e-10, atol=1e-7)
        assert p.nfft == 512 and p.bins == 257


def test_preemphasis_runs_descending():
    x = np.array([[1.0, 2.0, 4.0, 8.0]])
    np.testing.assert_allclose(R.preemphasis(x), [[0.03, 2.0 - 0.97, 4.0 - 1.94, 8.0 - 3.88]])


def test_mel_scale():
    assert abs(float(R.mel(1000.0)) - 1000.0) < 0.05  # 1000.0145: the HTK scale is anchored at 1 kHz
    np.testing.assert_allclose(R.mel_inv(R.mel([0.0, 440.0, 8000.0])), [0.0, 440.0, 8000.0], atol=1e-9)


@pytest.mark.parametrize("n_filters", [40, 80])
def test_filters_are_triangles_between_neighbour_centres(n_filters):
    bins = 257
    fb = R.filterbank(n_filters, bins, FS)
    e = R.filter_edges(n_filters, bins, FS)
    assert fb.shape == (n_filters, bins)
    assert (fb >= 0).all() and (fb <= 1 + 1e-12).all()
    assert e[0] == 0 and abs(e[-1] - (bins - 1)) < 1e-9
    i = np.arange(bins)
    for f in range(n_filters):
        nz = i[fb[f] > 0]
        # filter f lives strictly between the centres of filters f-1 and f+1 (= corners f and f+2)
        assert nz.size and nz.min() > e[f] and nz.max() < e[f + 2]
        assert fb[f].max() > 0.3  # the peak at corner f+1 is reached up to the bin spacing
    # neighbouring triangles cross-fade: the sum of two overlapping filters is 1 between their centres
    cover = fb.sum(0)[(i > e[1]) & (i < e[-2])]
    np.testing.assert_allclose(cover, 1.0, atol=1e-12)


@pytest.mark.parametrize("frame_ms,stride_ms", [(25, 10), (30, 10)])
def test_num_frames_at_the_edges(frame_ms, stride_ms):
    from wav2letter_b200.features import num_frames

    frame, stride = R.frame_samples(FS, frame_ms), R.frame_samples(FS, stride_ms)
    assert (frame, stride) == (16 * frame_ms, 160)
    for n, want in ((0, 0), (frame - 1, 0), (frame, 1), (frame + stride - 1, 1), (frame + stride, 2), (528000, 1 + (528000 - frame) // stride)):
        assert R.num_frames(n, FS, frame_ms, stride_ms) == want
        assert num_frames(n, FS, frame_ms, stride_ms) == want
    assert R.frame_samples(22050, 10) == 221  # 220.5 rounds up
    assert num_frames(10000, 22050, 25, 10) == 1 + (10000 - 551) // 221


class StreamingLocalNorm:
    """Line-by-line transcription of LocalNorm::run (recipes/streaming_convnets/inference/inference/module/nn/
    LocalNorm.cpp:50-106) in float32: std::accumulate(..., 0.0) sums in double and is stored as float; state (the
    per-frame sums of the last left_ctx + 1 frames) carries over between calls."""

    def __init__(self, feature_size, left_ctx):
        self.F, self.left = feature_size, left_ctx
        self.sum_buf, self.sq_buf = [], []

    def run(self, chunk):  # chunk [n, F] float32 -> [n, F]
        out = np.empty_like(chunk)
        for t in range(chunk.shape[0]):
            x = chunk[t]
            cur_sum = np.float32(sum(float(v) for v in x))
            cur_sq = np.float32(sum(float(v) * float(v) for v in x))
            self.sum_buf.append(cur_sum)
            self.sq_buf.append(cur_sq)
            total = len(self.sum_buf)
            total_sum = np.float32(sum(float(v) for v in self.sum_buf))
            total_sq = np.float32(sum(float(v) for v in self.sq_buf))
            mean = np.float32(total_sum / np.float32(total * self.F))
            std = np.float32(np.sqrt(np.float32(total_sq / np.float32(total * self.F)) - mean * mean))
            if std <= np.float32(1e-5):
                std = np.float32(1.0)
            out[t] = (x - mean) / std
            if total > self.left:
                self.sum_buf.pop(0)
                self.sq_buf.pop(0)
        return out


@pytest.mark.parametrize("left_ctx", [1, 7, 300])
def test_local_normalisation_matches_streaming_localnorm(left_ctx):
    rng = np.random.default_rng(left_ctx)
    T, F = 420, 40
    # log-mel-like values: a slowly drifting level per frame, spread over the filters
    f = (6.0 + 2.0 * np.sin(np.arange(T) / 37.0)[:, None] + rng.normal(0, 1.5, (T, F))).astype(np.float32)
    ln = StreamingLocalNorm(F, left_ctx)
    cuts = [0, 1, 17, 60, 61, 250, T]
    got = np.concatenate([ln.run(f[a:b]) for a, b in zip(cuts[:-1], cuts[1:])])
    np.testing.assert_allclose(R.normalize_local(f.astype(np.float64), left_ctx), got, atol=2e-4)


def test_utterance_normalisation_and_padding():
    rng = np.random.default_rng(3)
    fr = R.frame_samples(FS, 25)
    audio = [rng.normal(0, 800, 8000), np.zeros(4000), rng.normal(0, 800, fr - 1), rng.normal(0, 800, fr)]
    out = R.mfsc_batch(audio, [len(a) for a in audio], n_filters=40)
    assert out.shape == (4, 40, 48)
    f0 = out[0]
    assert abs(f0.mean()) < 1e-12 and abs(f0.std() - 1.0) < 1e-12
    assert (out[1] == 0).all()            # silence: log(max(0, 1)) = 0 everywhere, std 0 counts as 1
    assert (out[2] == 0).all()            # shorter than a frame: no frames
    assert (out[3, :, 1:] == 0).all() and abs(out[3, :, 0].mean()) < 1e-12   # exactly one frame
    assert np.isfinite(out).all()


def test_abi_prototypes_and_argument_errors():
    from wav2letter_b200 import capi

    lib = capi.lib
    for s in ("w2l_mfsc_num_frames", "w2l_mfsc_workspace_size", "w2l_mfsc"):
        assert s in capi.PROTOTYPES and hasattr(lib, s)
    one = ctypes.c_void_p(256)  # never dereferenced: validation fails first
    n = (ctypes.c_int32 * 2)(16000, 8000)
    need = lib.w2l_mfsc_workspace_size(2, 16000, FS, 25, 10, 80)
    assert need >= 2 * 100 * 516 * 4
    assert lib.w2l_mfsc_workspace_size(0, 16000, FS, 25, 10, 80) == 0

    def call(B=2, S=16000, fs=FS, fms=25, sms=10, F=80, left=0, T=98, ws_bytes=1 << 40, lengths=n):
        return lib.w2l_mfsc(None, B, S, one, lengths, fs, fms, sms, F, left, one, T, one, ws_bytes)

    assert call(B=0) == 1 and b"positive" in lib.w2l_last_error()
    assert call(B=-3) == 1
    assert call(F=0) == 1
    assert call(left=-1) == 1
    assert call(T=97) == 1                                      # shorter than the longest utterance
    assert call(lengths=(ctypes.c_int32 * 2)(16001, 0)) == 1    # longer than max_samples
    assert lib.w2l_mfsc(None, 2, 16000, one, None, FS, 25, 10, 80, 0, one, 98, one, 1 << 40) == 1
    assert call(fs=22050, S=22050, lengths=(ctypes.c_int32 * 2)(22050, 0), T=98) == 4   # stride 221 samples: not a TMA row
    assert b"multiple of 4" in lib.w2l_last_error()
    assert call(fms=200) == 4                                   # 3200-sample frames
    assert call(F=300) == 4
    assert call(ws_bytes=need - 1) == 2 and b"workspace" in lib.w2l_last_error()
    assert lib.w2l_mfsc_num_frames(-1, FS, 25, 10) == -1
    assert lib.w2l_mfsc_num_frames(400, FS, 0, 10) == -1
