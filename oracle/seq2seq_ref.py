"""float64 reference of the Seq2Seq criterion (DESIGN.md §9) -- TEST INFRASTRUCTURE ONLY (never imported by the product).

Plain torch float64 with gradients from autograd, following the restated flashlight 0.3 Seq2SeqCriterion of DESIGN.md §9:
embedding (startEmbedding, then E[y~_{u-1}]), R rounds of an S-layer GRU stack (gate order r, z, n; every layer from
hidden state 0; dropout after every layer but the stack's last) and key-value attention (keys x[.][:H], values
x[.][H:], scores q.k / sqrt(H) + soft window), h = q + context, then the output Linear, log-softmax and the
label-smoothed NLL summed over the non-pad rows.

Parameters come from the trainer's criterion arena in layout() order: E [N][H], startEmbedding [H], per round and layer
W_ih [3H][H], W_hh [3H][H], b_ih [3H], b_hh [3H], then W_o [N][H], b_o [N].  The random draws (substituted tokens,
dropout scales) are inputs: tests/seq2seq_reference.py reproduces the library's bit for bit.
"""
from __future__ import annotations

import math

import torch


def param_shapes(N: int, H: int, rounds: int = 1, layers: int = 1):
    shapes = [(N, H), (H,)]
    for _ in range(rounds * layers):
        shapes += [(3 * H, H), (3 * H, H), (3 * H,), (3 * H,)]
    return shapes + [(N, H), (N,)]


def unflatten(flat, layout, N: int, H: int, rounds: int = 1, layers: int = 1):
    """float64 leaf tensors (requires_grad) from the flat criterion arena and Trainer.layout(1)"""
    flat = torch.as_tensor(flat).detach().double().cpu()
    shapes = param_shapes(N, H, rounds, layers)
    assert len(layout) == len(shapes), (len(layout), len(shapes))
    out = []
    for (off, n, _), shp in zip(layout, shapes):
        assert n == math.prod(shp)
        out.append(flat[off:off + n].reshape(shp).clone().requires_grad_(True))
    return out


def flatten_grads(params, layout, total: int):
    g = torch.zeros(total, dtype=torch.float64)
    for p, (off, n, _) in zip(params, layout):
        g[off:off + n] = p.grad.reshape(-1)
    return g


def gru_layer(x, W_ih, W_hh, b_ih, b_hh, h0=None):
    """x [B,U,H] -> outputs [B,U,H] (cuDNN's GRU, gate order r, z, n), and the last state"""
    B, U, H = x.shape
    h = torch.zeros(B, H, dtype=x.dtype) if h0 is None else h0
    gi = x @ W_ih.T + b_ih
    outs = []
    for u in range(U):
        gh = h @ W_hh.T + b_hh
        r = torch.sigmoid(gi[:, u, :H] + gh[:, :H])
        z = torch.sigmoid(gi[:, u, H:2 * H] + gh[:, H:2 * H])
        n = torch.tanh(gi[:, u, 2 * H:] + r * gh[:, 2 * H:])
        h = (1 - z) * n + z * h
        outs.append(h)
    return torch.stack(outs, 1), h


def window(U: int, Tp: int, std: float):
    """w[u][t] = -(t - u T'/U)^2 / (2 std^2)"""
    u = torch.arange(U, dtype=torch.float64)[:, None]
    t = torch.arange(Tp, dtype=torch.float64)[None, :]
    return -((t - u * Tp / U) ** 2) / (2 * std * std)


def attention(q, x, win=None):
    """q [B,U,H], x [B,T',2H] -> q + context"""
    H = q.shape[-1]
    k, v = x[..., :H], x[..., H:]
    s = q @ k.transpose(1, 2) / math.sqrt(H)
    if win is not None:
        s = s + win
    return q + torch.softmax(s, -1) @ v


def logits(params, x, tokens, rounds=1, layers=1, window_std=0.0, dropout_scales=None):
    """tokens [B,U] the decoder inputs (N = startEmbedding); dropout_scales[k] [B,U,H] after layer k (None: none)"""
    E, start = params[0], params[1]
    N, H = E.shape
    B, U = tokens.shape
    tok = torch.as_tensor(tokens, dtype=torch.long)
    table = torch.cat([E, start[None, :]], 0)
    h = table[tok]
    win = window(U, x.shape[1], window_std) if window_std > 0 else None
    for r in range(rounds):
        cur = h
        for l in range(layers):
            k = r * layers + l
            W_ih, W_hh, b_ih, b_hh = params[2 + 4 * k: 6 + 4 * k]
            cur, _ = gru_layer(cur, W_ih, W_hh, b_ih, b_hh)
            if dropout_scales is not None and l + 1 < layers:
                cur = cur * torch.as_tensor(dropout_scales[k], dtype=torch.float64)
        h = attention(cur, x, win)
    W_o, b_o = params[-2], params[-1]
    return h @ W_o.T + b_o


def loss(params, x, y, pad: int, tokens, rounds=1, layers=1, window_std=0.0, labelsmooth=0.0, dropout_scales=None):
    """per-utterance loss [B]: sum over rows with y != pad of (1 - ls) (-log p_y) - (ls / N) sum_c log p_c"""
    o = logits(params, x, tokens, rounds, layers, window_std, dropout_scales)
    lp = torch.log_softmax(o, -1)
    y = torch.as_tensor(y, dtype=torch.long)
    N = lp.shape[-1]
    nll = -lp.gather(-1, y[..., None])[..., 0]
    row = (1 - labelsmooth) * nll - (labelsmooth / N) * lp.sum(-1)
    return (row * (y != pad)).sum(1)


def teacher_tokens(y, N: int):
    """decoder inputs without substitution: start, then y[:, :-1]"""
    y = torch.as_tensor(y, dtype=torch.long)
    return torch.cat([torch.full((y.shape[0], 1), N, dtype=torch.long), y[:, :-1]], 1)


@torch.no_grad()
def greedy(params, x, eos: int, maxlen: int, rounds=1, layers=1):
    """float64 greedy decode of each utterance: (tokens, gaps) with gaps[i] the margin between the top two logits of
    step i (the decode is only determined where it is not tiny)"""
    E, start = params[0], params[1]
    H = E.shape[1]
    out = []
    for b in range(x.shape[0]):
        xb = x[b:b + 1]
        inp = start[None, None, :]
        states = [None] * (rounds * layers)
        toks, gaps = [], []
        for _ in range(maxlen):
            h = inp
            for r in range(rounds):
                cur = h
                for l in range(layers):
                    k = r * layers + l
                    W_ih, W_hh, b_ih, b_hh = params[2 + 4 * k: 6 + 4 * k]
                    cur, states[k] = gru_layer(cur, W_ih, W_hh, b_ih, b_hh, states[k])
                h = attention(cur, xb)
            o = (h @ params[-2].T + params[-1])[0, 0]
            top = torch.topk(o, 2).values
            gaps.append(float(top[0] - top[1]))
            t = int(torch.argmax(o))
            if t == eos:
                break
            toks.append(t)
            inp = E[t][None, None, :]
        out.append((toks, gaps))
    return out
