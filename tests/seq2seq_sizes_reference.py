"""float64 reference of the Seq2Seq criterion on padded batches (DESIGN.md §9 "Padded batches") -- TEST INFRASTRUCTURE ONLY.

  frame_counts   T'_b = ceil(d_b T' / max d) clamped to [1, T'], and which utterances the sizes reject
  attention      key-value attention of utterance b over its frames t < T'_b; nothing past them is read
  loss           the criterion's per-utterance loss with per-utterance frame counts and target sizes (the window centred
                 at u T'_b / U_b), built on oracle/seq2seq_ref.py's GRU layer
  greedy         the greedy decode of a padded batch in lock step, each utterance over its own frames
  model_step     tests/seq2seq_beam_reference.py's step function over x[b, :T'_b]

The window centre is computed in float64 here, as oracle/seq2seq_ref.py computes it; the kernels compute it in fp32.
With every T'_b = T' and U_b = U each function gives the unsized oracle's values exactly.
"""
import math

import torch

import seq2seq_beam_reference as beamref
from oracle import seq2seq_ref as ref


def frame_counts(durations, Tp: int, target_sizes=None, U: int | None = None):
    """(tps, ups, bad) lists of B: T'_b from the input frame counts (None: T'), U_b from the target sizes (None: U), and
    bad[b] when a duration is <= 0 or not whole, no duration is positive, or a target size lies outside [1, U]"""
    B = len(durations) if durations is not None else len(target_sizes)
    tps, ups, bad = [Tp] * B, [U] * B, [False] * B
    if durations is not None:
        ok = [float(d) > 0 and float(d) == math.floor(float(d)) and math.isfinite(float(d)) for d in durations]
        dmax = max([float(d) for d, o in zip(durations, ok) if o], default=0.0)
        for b, d in enumerate(durations):
            if ok[b] and dmax > 0:
                tps[b] = int(min(max(math.ceil(float(d) * Tp / dmax), 1), Tp))
            else:
                bad[b] = True  # its bound stays T'
    if target_sizes is not None:
        for b, v in enumerate(target_sizes):
            if 1 <= int(v) <= U:
                ups[b] = int(v)
            else:
                bad[b] = True
    return tps, ups, bad


def window(U: int, Tp: int, tps, ups, std: float):
    """[B,U,T'] w[b][u][t] = -(t - u T'_b / U_b)^2 / (2 std^2)"""
    u = torch.arange(U, dtype=torch.float64)[None, :, None]
    t = torch.arange(Tp, dtype=torch.float64)[None, None, :]
    tb = torch.as_tensor(tps, dtype=torch.float64)[:, None, None]
    ub = torch.as_tensor(ups, dtype=torch.float64)[:, None, None]
    return -((t - u * tb / ub) ** 2) / (2 * std * std)


def mask(tps, Tp: int):
    """[B,1,T'] True on the frames of each utterance"""
    return torch.arange(Tp)[None, None, :] < torch.as_tensor(tps)[:, None, None]


def attention(q, x, tps, win=None):
    """q [B,U,H], x [B,T',2H] -> q + context over t < T'_b; frames past T'_b are replaced by 0 before use, so NaN there
    reaches neither the result nor the gradient"""
    H = q.shape[-1]
    m = mask(tps, x.shape[1])
    xm = torch.where(m.transpose(1, 2), x, torch.zeros((), dtype=x.dtype))
    k, v = xm[..., :H], xm[..., H:]
    s = q @ k.transpose(1, 2) / math.sqrt(H)
    if win is not None:
        s = s + win
    s = torch.where(m, s, torch.tensor(-math.inf, dtype=s.dtype))
    return q + torch.softmax(s, -1) @ v


def logits(params, x, tokens, tps, ups, rounds=1, layers=1, window_std=0.0, dropout_scales=None):
    """oracle/seq2seq_ref.py's logits with per-utterance frame counts and window targets"""
    E, start = params[0], params[1]
    B, U = tokens.shape
    table = torch.cat([E, start[None, :]], 0)
    h = table[torch.as_tensor(tokens, dtype=torch.long)]
    win = window(U, x.shape[1], tps, ups, window_std) if window_std > 0 else None
    for r in range(rounds):
        cur = h
        for l in range(layers):
            k = r * layers + l
            W_ih, W_hh, b_ih, b_hh = params[2 + 4 * k: 6 + 4 * k]
            cur, _ = ref.gru_layer(cur, W_ih, W_hh, b_ih, b_hh)
            if dropout_scales is not None and l + 1 < layers:
                cur = cur * torch.as_tensor(dropout_scales[k], dtype=torch.float64)
        h = attention(cur, x, tps, win)
    return h @ params[-2].T + params[-1]


def loss(params, x, y, pad: int, tokens, tps, ups, rounds=1, layers=1, window_std=0.0, labelsmooth=0.0, dropout_scales=None):
    """per-utterance loss [B] as oracle/seq2seq_ref.py's loss; target sizes only move the window"""
    o = logits(params, x, tokens, tps, ups, rounds, layers, window_std, dropout_scales)
    lp = torch.log_softmax(o, -1)
    y = torch.as_tensor(y, dtype=torch.long)
    N = lp.shape[-1]
    nll = -lp.gather(-1, y[..., None])[..., 0]
    row = (1 - labelsmooth) * nll - (labelsmooth / N) * lp.sum(-1)
    return (row * (y != pad)).sum(1)


@torch.no_grad()
def greedy(params, x, tps, eos: int, maxlen: int, rounds=1, layers=1):
    """the greedy decode of the whole padded batch in lock step, one masked attention per step: [(tokens, gaps)] per
    utterance as oracle/seq2seq_ref.py's greedy returns them"""
    E, start = params[0], params[1]
    B, H = x.shape[0], E.shape[1]
    inp = start[None, None, :].expand(B, 1, H)
    states = [None] * (rounds * layers)
    out = [([], []) for _ in range(B)]
    live = [True] * B
    for _ in range(maxlen):
        h = inp
        for r in range(rounds):
            cur = h
            for l in range(layers):
                k = r * layers + l
                W_ih, W_hh, b_ih, b_hh = params[2 + 4 * k: 6 + 4 * k]
                cur, states[k] = ref.gru_layer(cur, W_ih, W_hh, b_ih, b_hh, states[k])
            h = attention(cur, x, tps)
        o = (h @ params[-2].T + params[-1])[:, 0]
        nxt = []
        for b in range(B):
            t = int(torch.argmax(o[b]))
            if live[b]:
                top = torch.topk(o[b], 2).values
                out[b][1].append(float(top[0] - top[1]))
                if t == eos:
                    live[b] = False
                else:
                    out[b][0].append(t)
            nxt.append(E[t] if t != eos else E[0])
        if not any(live):
            break
        inp = torch.stack(nxt)[:, None, :]
    return out


def model_step(params, x, Tb: int, rounds=1, layers=1):
    """(step, init) for seq2seq_beam_reference.beam: the decoder of one utterance x [1,T',2H] over its first Tb frames"""
    return beamref.model_step(params, x[:, :Tb], rounds, layers)
