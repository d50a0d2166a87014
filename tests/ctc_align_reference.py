"""NumPy float32 restatement of the CTC Viterbi-with-target contract (w2l_ctc_viterbi_target in include/w2l_b200.h).

Scores are the raw activations; alpha_t[s] = fp32(max(alpha_{t-1}[s], alpha_{t-1}[s-1], alpha_{t-1}[s-2] if the skip
is allowed) + e_t[z_s]); predecessors are taken in the order s, s-1, s-2 and a later one wins only if strictly greater;
the end state is S-1 unless alpha_{T-1}[S-2] > alpha_{T-1}[S-1].  A target that needs more than T frames, or holds a
label outside [0, N-1), gives -1 for the whole utterance.  The batch is walked together (one [B, S_max] row per frame)."""
import numpy as np

NEG = np.float32(-np.inf)


def target_size(row):
    nz = np.nonzero(np.asarray(row) >= 0)[0]
    return int(nz[-1]) + 1 if len(nz) else 0


def ctc_viterbi_target(emis, target, return_score=False):
    """emis float32 [B,T,N], target int32 [B,L] (-1 padded) -> (path [B,T], state [B,T]) int32 (+ the float32 score
    alpha_{T-1}[end] per utterance, NaN where there is none)"""
    emis = np.asarray(emis, np.float32)
    target = np.asarray(target, np.int32).reshape(emis.shape[0], -1)
    B, T, N = emis.shape
    blank = N - 1
    path = np.full((B, T), -1, np.int32)
    state = np.full((B, T), -1, np.int32)
    score = np.full(B, np.nan, np.float32)
    rows = []
    for b in range(B):
        y = target[b, : target_size(target[b])]
        if np.any(y < 0) or np.any(y >= N - 1) or len(y) + int(np.sum(y[1:] == y[:-1])) > T:
            continue
        rows.append((b, y))
    if not rows:
        return (path, state, score) if return_score else (path, state)
    bs = np.array([b for b, _ in rows])
    S = np.array([2 * len(y) + 1 for _, y in rows])
    Smax = int(S.max())
    z = np.full((len(rows), Smax), blank, np.int64)
    skip = np.zeros((len(rows), Smax), bool)
    live = np.arange(Smax)[None, :] < S[:, None]
    for r, (_, y) in enumerate(rows):
        z[r, 1 : 2 * len(y) : 2] = y
        skip[r, 3 : 2 * len(y) : 2] = y[1:] != y[:-1]
    e = lambda t: emis[bs[:, None], t, z]  # [R, Smax] float32
    a = np.full((len(rows), Smax), NEG, np.float32)
    a[:, 0] = e(0)[:, 0]
    if Smax > 1:
        a[S > 1, 1] = e(0)[S > 1, 1]
    bp = np.zeros((T, len(rows), Smax), np.int8)
    ninf1 = np.full((len(rows), 1), NEG, np.float32)
    ninf2 = np.full((len(rows), 2), NEG, np.float32)
    for t in range(1, T):
        p1 = np.concatenate([ninf1, a], axis=1)[:, :Smax]
        p2 = np.where(skip, np.concatenate([ninf2, a], axis=1)[:, :Smax], NEG)
        best = a
        code = np.zeros(a.shape, np.int8)
        m = p1 > best
        best = np.where(m, p1, best)
        code[m] = 1
        m = p2 > best
        best = np.where(m, p2, best)
        code[m] = 2
        a = np.where(live, (best + e(t)).astype(np.float32), NEG)
        bp[t] = code
    for r, (b, y) in enumerate(rows):
        n = S[r]
        s = n - 2 if n > 1 and a[r, n - 2] > a[r, n - 1] else n - 1
        score[b] = a[r, s]
        for t in range(T - 1, -1, -1):
            state[b, t] = s
            path[b, t] = z[r, s]
            if t > 0:
                s -= bp[t, r, s]
    return (path, state, score) if return_score else (path, state)


def collapse(path, blank):
    """CTC decoding of one frame path: drop repeats, then blanks"""
    out, prev = [], None
    for p in path:
        if p != prev and p != blank:
            out.append(int(p))
        prev = p
    return out
