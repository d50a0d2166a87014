"""float64 beam search of the Seq2Seq criterion (DESIGN.md §9 "Beam search") -- TEST INFRASTRUCTURE ONLY.

  beam         the search over a generic step function, so that synthetic log-prob tables and the model both drive it;
               returns the n-best list and every decision margin
  model_step   the step function of the criterion's decoder for one utterance, built on oracle/seq2seq_ref.py's GRU
               layer and attention
"""
import numpy as np
import torch

from oracle.seq2seq_ref import attention, gru_layer


def beam(step, init, K: int, maxlen: int, eos: int):
    """float64 beam search of DESIGN.md §9 over a generic step function: step(state) -> (logp [N], cont), with cont(token)
    the state after that token; init the start state (the model: startEmbedding and zero GRU states; a synthetic table:
    the empty prefix).  Returns (hyps, margins): hyps [(score, path)] as the search returns them, margins every decision
    gap -- consecutive sorted candidates at each rank the walk reads and at the rank after it, consecutive completions up
    to the one the K-cap drops, and the early-stop comparison.  A search run in another precision takes the same
    decisions while its score errors stay below min(margins) / 2."""
    live = [(0.0, [], init)]
    comps, margins = [], []
    for _ in range(maxlen):
        cand, conts = [], []
        for h, (s, _path, st) in enumerate(live):
            lp, cont = step(st)
            lp = np.asarray(lp, np.float64)
            N = len(lp)
            conts.append(cont)
            cand += [(s + float(lp[c]), h * N + c) for c in range(N)]
        cand.sort(key=lambda e: (-e[0], e[1]))
        new, last = [], 0
        for j, (sc, flat) in enumerate(cand):
            h, c = divmod(flat, N)
            last = j
            if c == eos:
                if j < K:
                    comps.append((sc, list(live[h][1])))
            else:
                new.append((sc, live[h][1] + [c], h, c))
                if len(new) == K:
                    break
        margins += [cand[r][0] - cand[r + 1][0] for r in range(min(last + 1, len(cand) - 1))]
        live = [(sc, path, conts[h](c)) for sc, path, h, c in new]
        if len(comps) >= K:
            comps.sort(key=lambda e: -e[0])  # stable: equal scores keep their completion order
            margins += [comps[r][0] - comps[r + 1][0] for r in range(min(K, len(comps) - 1))]
            comps = comps[:K]
            margins.append(abs(comps[K - 1][0] - live[0][0]))
            if comps[K - 1][0] > live[0][0]:
                break
    hyps = comps if comps else [(sc, path) for sc, path, _st in live]
    return hyps, margins


def model_step(params, x, rounds=1, layers=1):
    """(step, init) for beam(): the decoder of one utterance x [1,T',2H] in eval mode, without the window"""
    E, start = params[0], params[1]
    W_o, b_o = params[-2], params[-1]

    def step(state):
        inp, states = state
        states = list(states)
        with torch.no_grad():
            h = inp[None, None, :]
            for r in range(rounds):
                cur = h
                for l in range(layers):
                    k = r * layers + l
                    W_ih, W_hh, b_ih, b_hh = params[2 + 4 * k: 6 + 4 * k]
                    cur, states[k] = gru_layer(cur, W_ih, W_hh, b_ih, b_hh, states[k])
                h = attention(cur, x)
            lp = torch.log_softmax((h @ W_o.T + b_o)[0, 0], -1).numpy()
        return lp, lambda t: (E[t].detach(), states)

    return step, (start.detach(), [None] * (rounds * layers))
