"""NumPy fp32 model of the streaming acoustic model's criterion path for ASG / LinSeg (w2l_stream_run_path,
DESIGN.md §4 "Streaming acoustic model"): the FCC Viterbi recursion carried across calls, the convergence rule and the
forced commit.

One slot holds alpha (never re-centred), its first-frame flag and the backpointers of its pending (uncommitted) frames.
A call advances alpha over its new frames with fp32 adds, candidates j ascending and the first maximum winning, then
traces every state back through the pending frames to the newest frame at which all states agree and commits every
frame up to it.  On finish it commits the rest along the first-maximum end state; otherwise, when more than
`max_pending` frames are pending, it commits the oldest ones along that state's path and counts them as forced."""
import numpy as np


class CarriedViterbi:
    def __init__(self, trans, max_pending: int = 1024):
        self.trans = np.ascontiguousarray(trans, dtype=np.float32)  # [N][N]: trans[to][from]
        self.N = self.trans.shape[0]
        self.max_pending = int(max_pending)
        self.alpha = None
        self.bp = []  # per pending frame: the previous state of every state (the first frame's is never read)
        self.committed = 0
        self.forced = 0

    def _step(self, e):
        if self.alpha is None:
            self.alpha = e.copy()
            self.bp.append(np.zeros(self.N, np.int64))
            return
        cand = self.alpha[None, :] + self.trans  # [to][from], fp32
        arg = np.argmax(cand, axis=1)  # the first maximum, as the strict '>' over ascending j
        self.alpha = (cand[np.arange(self.N), arg] + e).astype(np.float32)
        self.bp.append(arg)

    def _commit(self, count, last):
        labels = np.zeros(count, np.int32)
        st = int(last)
        for k in range(count - 1, -1, -1):
            labels[k] = st
            if k > 0:
                st = int(self.bp[k][st])
        del self.bp[:count]
        return labels

    def run(self, emis, finish: bool = False):
        """emis [f, N]: the call's new frames.  Returns (labels committed in this call, the stream frame index of the
        first of them, forced frames so far): the {path, path_info} of w2l_stream_run_path for this stream."""
        for e in np.asarray(emis, np.float32).reshape(-1, self.N):
            self._step(e)
        out = [np.zeros(0, np.int32)]
        pos = np.arange(self.N)
        for k in range(len(self.bp) - 1, -1, -1):
            if (pos == pos[0]).all():
                out.append(self._commit(k + 1, pos[0]))
                break
            if k == 0:
                break
            pos = self.bp[k][pos]
        P = len(self.bp)
        if P and (finish or P > self.max_pending):
            count = P if finish else P - self.max_pending
            st = int(np.argmax(self.alpha))
            for k in range(P - 1, count - 1, -1):
                st = int(self.bp[k][st])
            if not finish:
                self.forced += count
            out.append(self._commit(count, st))
        labels = np.concatenate(out)
        first = self.committed
        self.committed += len(labels)
        return labels, first, self.forced

    @property
    def pending(self) -> int:
        return len(self.bp)


def tied_forever(N: int, frames: int):
    """emissions [frames, N] and transitions [N][N] under which states 0 and 1 keep the same score at every frame and
    each keeps its own predecessor, so their paths never meet: only finish or the forced commit can commit a frame.
    Every value is a small integer, so every sum is exact in fp32."""
    trans = np.full((N, N), -8.0, np.float32)
    np.fill_diagonal(trans, 0.0)
    emis = np.full((frames, N), -64.0, np.float32)
    emis[:, :2] = 1.0
    return emis, trans
