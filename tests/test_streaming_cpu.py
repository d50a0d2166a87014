"""The streaming acoustic model's frame bookkeeping (w2l_stream_plan, host only) against a NumPy simulation of the
in-tree inference library's convolution buffers (inference/module/nn/backend/fbgemm/Conv1dFbGemm.cpp): start writes
pad_left zero frames, run appends the new frames and, with avail >= kw frames held, emits (avail - kw) / stride + 1
frames and consumes stride frames per output, finish appends pad_right zero frames and runs.  Every layer of the
BASELINE streaming arch, over random chunk sequences; no GPU needed."""
import numpy as np
import pytest

from wav2letter_b200 import archs

ARCH = archs.streaming_tds()


def conv_specs(arch_text):
    """(kw, stride, pad_left, pad_right) of every convolution, read from the arch text"""
    out, pend = [], None
    for line in arch_text.splitlines():
        p = line.split()
        if not p:
            continue
        if p[0] == "PD":
            pend = (int(p[2]), int(p[3]))
        elif p[0] == "C2":
            k, s = int(p[3]), int(p[5])
            pl, pr = pend if pend else ((k - s + 1) // 2,) * 2
            out.append((k, s, pl, pr))
            pend = None
        elif p[0] == "TDS":
            k, r = int(p[2]), int(p[6])
            out.append((k, 1, k - 1 - r, r))
    return out


class ConvBuffer:
    """Conv1dFbGemm's input buffer; frames carry their index in the layer's padded input (-1: padding)"""

    def __init__(self, kw, stride, pl, pr):
        self.kw, self.stride, self.pr = kw, stride, pr
        self.buf = np.full(pl, -1, dtype=np.int64)
        self.seen = 0

    def run(self, n_new, finish=False):
        self.buf = np.concatenate([self.buf, np.arange(self.seen, self.seen + n_new)])
        self.seen += n_new
        if finish:
            self.buf = np.concatenate([self.buf, np.full(self.pr, -1, dtype=np.int64)])
        if len(self.buf) < self.kw:
            return 0
        n_out = (len(self.buf) - self.kw) // self.stride + 1
        self.buf = self.buf[n_out * self.stride:]
        return n_out


def simulate(specs, chunks, finish=True):
    convs = [ConvBuffer(*s) for s in specs]
    outs, tails = [], []
    for k, n in enumerate(chunks):
        row_o, row_t = [], []
        for c in convs:
            n = c.run(n, finish and k == len(chunks) - 1)
            row_o.append(n)
            row_t.append(len(c.buf))
        outs.append(row_o)
        tails.append(row_t)
    return np.array(outs, dtype=np.int64).reshape(len(chunks), len(specs)), np.array(tails, dtype=np.int64).reshape(len(chunks), len(specs))


def offline_frames(specs, T):
    for k, s, pl, pr in specs:
        T = (T + pl + pr - k) // s + 1 if T + pl + pr >= k else 0
    return T


def test_conv_specs_are_the_arch_s():
    from wav2letter_b200 import streaming

    specs, _, _ = streaming.plan(ARCH, 80, 10000, [])
    assert specs == conv_specs(ARCH)
    assert len(specs) == 4 + 2 + 3 + 4 + 5


@pytest.mark.parametrize("seed", range(6))
def test_bookkeeping_matches_the_buffer_rule(seed):
    from wav2letter_b200 import streaming

    rng = np.random.default_rng(seed)
    specs = conv_specs(ARCH)
    for trial in range(20):
        n_calls = int(rng.integers(1, 30))
        chunks = [int(x) for x in rng.integers(0, [1, 8, 60, 200][trial % 4] + 1, n_calls)]
        finish = trial % 5 != 4
        _, out, tails = streaming.plan(ARCH, 80, 10000, chunks, finish)
        ref_out, ref_tails = simulate(specs, chunks, finish)
        np.testing.assert_array_equal(out, ref_out)
        np.testing.assert_array_equal(tails, ref_tails)
        for (k, s, pl, pr), t in zip(specs, tails.T):
            assert t.max() <= max(k - 1, pl)
        if finish:  # the split into chunks does not matter: the whole utterance's frame count
            assert out[:, -1].sum() == offline_frames(specs, sum(chunks))


def test_plan_rejects_non_streaming_archs_with_the_export_text():
    from wav2letter_b200 import W2LError, streaming

    with pytest.raises(W2LError, match="unsupported LayerNorm axis"):
        streaming.plan("V -1 NFEAT 1 0\nC2 1 4 5 1 2 1 -1 -1\nR\nLN 3\nV 0 320 1 0\nRO 1 0 3 2\nL 320 NLABEL\n", 80, 8, [10])
    with pytest.raises(W2LError, match="lNormIncludeTime"):
        streaming.plan("V -1 NFEAT 1 0\nC2 1 4 5 1 1 1 0 0\nTDS 4 5 80 0.0 0 1 1\nL 320 NLABEL\n", 80, 8, [10])
    with pytest.raises(W2LError, match="negative"):
        streaming.plan(ARCH, 80, 10, [5, -1])
