"""numpy emulation of the arithmetic formulation the CUDA ASG kernels use (fp32 where the
kernels use fp32).  This is NOT the product and NOT the oracle: it exists so that the kernel
math (scaling bookkeeping, meet-in-the-middle junction, gradient identities) can be checked
against the oracle on the CPU-only dev box before a GPU round trip.  See DESIGN.md §kernels.
"""
import numpy as np

F = np.float32


def pow2_scale(mx, damp=0):
    """2^-(exponent(mx) >> damp) built from the exponent bits (exact), clamp like the kernel."""
    bits = np.float32(mx).view(np.int32)
    k = int((bits >> 23) & 0xFF) - 127
    k = max(-126, min(126, k)) >> damp
    return F(2.0) ** F(-k), k


def fcc_emulate(e, tr, alpha_damp=1, return_exponents=False):
    """Linear-domain FCC alpha/beta with lagged power-of-two rescaling.
    returns logZ, gamma[T,N], xi_sum[N,N]"""
    T, N = e.shape
    tmax = tr.max()
    M = np.exp((tr - tmax).astype(F)).astype(F)  # M[i][j]
    m = e.max(axis=1)
    X = np.exp((e - m[:, None]).astype(F)).astype(F)
    A = np.zeros((T, N), F)
    sA = np.ones(T, F)
    a = X[0].copy()
    A[0] = a
    ksum = 0
    s = F(1.0)
    for t in range(1, T):
        v = a  # a_{t-1}
        acc = (M @ v).astype(F)
        mx = v.max()
        with np.errstate(over="ignore", under="ignore"):
            a = (X[t] * s) * acc
        A[t] = a
        sA[t] = s
        ksum += -int(np.log2(s))
        s, _ = pow2_scale(mx, alpha_damp)  # applied at the NEXT step from |a_{t-1}|: lag two, damped
    if return_exponents:
        with np.errstate(divide="ignore"):
            return np.log2(A.max(axis=1))
    logZ = float(m.astype(np.float64).sum()) + (T - 1) * float(tmax) + np.log(2.0) * ksum + np.log(
        float(a.astype(np.float64).sum()))
    Bh = np.zeros((T, N), F)
    bh = np.ones(N, F)
    Bh[T - 1] = bh
    s = F(1.0)
    for t in range(T - 2, -1, -1):
        u = bh * (X[t + 1] * s)
        mx = u.max()
        bh = (M.T @ u).astype(F)
        Bh[t] = bh
        s, _ = pow2_scale(mx)
    g = A * Bh
    gs = g.sum(axis=1)
    gamma = g / gs[:, None]
    xi = np.zeros((N, N), F)
    for t in range(1, T):
        w = X[t] * Bh[t] * (sA[t] / gs[t])
        xi += np.outer(w, A[t - 1])
    xi *= M
    return logZ, gamma, xi


def lse2(a, b):
    m = np.maximum(a, b)
    n = np.minimum(a, b)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = m + np.log1p(np.exp((n - m).astype(F))).astype(F)
    return np.where(n == -np.inf, m, r).astype(F)


def fac_emulate(e, y, tr):
    """ROUND-1 formulation (kept as an independent fp32 cross-check of the oracle; the kernels no longer use it):
    log-domain FAC, alpha from t=0 and beta from t=T-1 meeting at h=T//2, per-step
    re-centring by the band max, gamma = xi_stay + xi_adv, renormalised per frame.  returns logZ, G[T,N], dtrans[N,N]"""
    T, N = e.shape
    L = len(y)
    NI = F(-np.inf)
    s1 = tr[y, y].astype(F)
    s2 = np.concatenate([[NI], tr[y[1:], y[:-1]]]).astype(F)
    G = np.zeros((T, N), np.float64)
    dtr = np.zeros((N, N), np.float64)
    if T == 1:
        G[0, y[0]] = 1.0
        return float(e[0, y[0]]), G, dtr
    h = T // 2

    def band(t):
        return max(0, L - (T - t)), min(t, L - 1)

    def mask(row, t):
        lo, hi = band(t)
        out = np.full(L, NI, F)
        out[lo:hi + 1] = row[lo:hi + 1]
        return out

    alpha = np.full((T, L), NI, F)
    cA = np.zeros(T, np.float64)
    row = np.full(L, NI, F)
    row[0] = e[0, y[0]]
    alpha[0] = row
    C = 0.0

    def alpha_step(prev, t, C):
        d = prev.max()
        C += float(d)
        stay = prev + (s1 - d)
        adv = np.concatenate([[NI], prev[:-1]]) + (s2 - d)
        new = mask(e[t, y] + lse2(stay, adv), t)
        return new.astype(F), C

    for t in range(1, h):
        row, C = alpha_step(row, t, C)
        alpha[t] = row
        cA[t] = C
    beta = np.full((T, L), NI, F)
    cB = np.zeros(T, np.float64)
    rb = np.full(L, NI, F)
    rb[L - 1] = e[T - 1, y[L - 1]]
    beta[T - 1] = rb
    Cb = 0.0

    def beta_step(nxt, t, Cb):
        d = nxt.max()
        Cb += float(d)
        stay = nxt + (s1 - d)
        adv = np.concatenate([nxt[1:], [NI]]) + (np.concatenate([s2[1:], [NI]]) - d)
        new = mask(e[t, y] + lse2(stay, adv), t)
        return new.astype(F), Cb

    for t in range(T - 2, h - 1, -1):
        rb, Cb = beta_step(rb, t, Cb)
        beta[t] = rb
        cB[t] = Cb
    # junction at t = h
    prevA = row
    CA_prev = C
    row, C = alpha_step(row, h, C)
    alpha[h] = row
    cA[h] = C
    q = row + beta[h] - e[h, y]
    qm = q.max()
    tot = np.exp((q - qm).astype(F)).astype(F).sum(dtype=np.float64)
    logZ = cA[h] + cB[h] + float(qm) + np.log(tot)
    gam = np.exp((q - qm).astype(F)) / F(tot)
    np.add.at(G[h], y, gam)
    ds1 = np.zeros(L, np.float64)
    ds2 = np.zeros(L, np.float64)
    rn = {}  # per-frame normalisers 1/sum_l gamma_t[l]; the kernel applies them with a lag of two steps

    # group A: t = h+1 .. T-1
    for t in range(h + 1, T):
        prev = row
        Cp = C
        row, C = alpha_step(row, t, C)
        K = F(Cp + cB[t] - logZ)
        with np.errstate(invalid="ignore"):
            xs = np.exp((prev + s1 + beta[t] + K).astype(F))
            xa = np.exp((np.concatenate([[NI], prev[:-1]]) + s2 + beta[t] + K).astype(F))
        xs = np.nan_to_num(xs, nan=0.0)
        xa = np.nan_to_num(xa, nan=0.0)
        lag = rn.get(t - 2, 1.0) if t - 2 > h else 1.0
        ds1 += xs * lag
        ds2 += xa * lag
        tot = float((xs + xa).sum(dtype=np.float64))
        rn[t] = 1.0 / tot if tot > 0 else 0.0
        np.add.at(G[t], y, (xs + xa) * rn[t])
    rn = {}
    # group B: t = h-1 .. 0 (transitions t -> t+1)
    for t in range(h - 1, -1, -1):
        nxt = rb
        Cn = Cb
        rb, Cb = beta_step(rb, t, Cb)
        K = F(cA[t] + Cn - logZ)
        at = alpha[t]
        with np.errstate(invalid="ignore"):
            xs = np.exp((at + s1 + nxt + K).astype(F))
            xa = np.exp((at + np.concatenate([s2[1:], [NI]]) + np.concatenate([nxt[1:], [NI]]) + K).astype(F))
        xs = np.nan_to_num(xs, nan=0.0)
        xa = np.nan_to_num(xa, nan=0.0)
        lag = rn.get(t + 2, 1.0)
        ds1 += xs * lag
        ds2[1:] += xa[:-1] * lag
        tot = float((xs + xa).sum(dtype=np.float64))
        rn[t] = 1.0 / tot if tot > 0 else 0.0
        np.add.at(G[t], y, (xs + xa) * rn[t])
    np.add.at(dtr, (y, y), ds1)
    np.add.at(dtr, (y[1:], y[:-1]), ds2[1:])
    return logZ, G, dtr


# ------------------------------------------------------------------------------------------------------------------
# Round-2 formulation of the FAC recursions (criterion_asg.cu: fac_chain / asg_fac_grad_kernel): log2 domain, scores
# normalised by the frame maximum and the global transition maximum, lg2(1.25 * (1 + r)) with the constant folded into the
# transition scores, P consecutive positions per lane, re-centring every kRc frames either with ONE offset per row (the
# first version) or with one offset PER LANE (what the kernels do).  exp2 / log2 are exact here (float64, rounded to
# float32): the MUFU table error is a separate effect (DESIGN.md, ASG accuracy).
# ------------------------------------------------------------------------------------------------------------------
LOG2E = 1.4426950408889634
NEG = F(-1.0e30)
LG_SCALE = F(1.25)
LG_SHIFT = F(0.32192809488736235)


def _lse2_log2(a, b):
    mx = np.maximum(a, b)
    mn = np.minimum(a, b)
    d = (mn - mx).astype(F)
    r = np.exp2(d.astype(np.float64)).astype(F)
    q = (r * LG_SCALE + LG_SCALE).astype(F)
    return (mx + np.log2(q.astype(np.float64)).astype(F)).astype(F)


def fac_chain_emulate(e, y, tr, offsets="lane", P=8, kRc=2):
    """posteriors gamma[T][L] and log-partition (natural log) of the forced alignment, float32 arithmetic of the round-2
    kernels.  offsets: 'lane' (one re-centring offset per lane of P positions) or 'row' (one per row)."""
    T, N = e.shape
    L = len(y)
    e64 = e.astype(np.float64)
    m = e64.max(1, keepdims=True)
    z = ((e64 - m) * LOG2E).astype(F)
    tmax = float(tr.max())
    s1 = ((tr[y, y].astype(np.float64) - tmax) * LOG2E).astype(F) - LG_SHIFT
    s2a = np.full(L, NEG, F)
    s2a[1:] = ((tr[y[1:], y[:-1]].astype(np.float64) - tmax) * LOG2E).astype(F) - LG_SHIFT
    s2b = np.full(L, NEG, F)
    s2b[:-1] = s2a[1:]
    nl = (L + P - 1) // P
    lane = np.arange(L) // P

    def walk(beta):
        v = np.full(L, NEG, F)
        C = np.zeros(nl if offsets == "lane" else 1, np.float64)
        off = np.zeros_like(C)
        pend = np.full(C.shape, float(NEG))
        rows = np.zeros((T, L), np.float64)
        if not beta:
            v[0] = z[0, y[0]]
        else:
            v[L - 1] = z[T - 1, y[L - 1]]

        def total():
            return v.astype(np.float64) + (C[lane] if offsets == "lane" else C[0])

        rows[T - 1 if beta else 0] = total()
        for t in (range(T - 2, -1, -1) if beta else range(1, T)):
            if not beta:
                nb = np.concatenate(([NEG], v[:-1]))
                if offsets == "lane":  # the value crossing a lane boundary is re-based by the offset difference
                    nb = (nb + np.concatenate(([0.0], C[lane[:-1]] - C[lane[1:]])).astype(F)).astype(F)
                v = (z[t, y] + _lse2_log2((v + s1).astype(F), (nb + s2a).astype(F))).astype(F)
            else:
                nb = np.concatenate((v[1:], [NEG]))
                if offsets == "lane":
                    nb = (nb + np.concatenate((C[lane[1:]] - C[lane[:-1]], [0.0])).astype(F)).astype(F)
                v = (z[t, y] + _lse2_log2((v + s1).astype(F), (nb + s2b).astype(F))).astype(F)
            # lagged re-centring: the maximum taken at one frame is subtracted after the next one; the maximum is put at
            # +off, half of what it lost over the last period
            apply_phase = (t % kRc) == (kRc - 1 if beta else 0)
            measure_phase = (t % kRc) == (0 if beta else kRc - 1)
            if apply_phase:
                for j in range(len(C)):
                    sl = slice(j * P, (j + 1) * P) if offsets == "lane" else slice(0, L)
                    if pend[j] > -1e29:
                        off_new = min(max(0.5 * (off[j] - pend[j]), 0.0), 48.0)
                        mm = F(pend[j] - off_new)
                        off[j] = off_new
                        v[sl] = (v[sl] - mm).astype(F)
                        C[j] += float(mm)
                    elif offsets == "lane":  # a lane that holds nothing yet follows its neighbour's offset
                        jn = j + 1 if beta else j - 1
                        if 0 <= jn < len(C):
                            v[sl] = (v[sl] - F(C[jn] - C[j])).astype(F)
                            C[j] = C[jn]
            if measure_phase:
                for j in range(len(C)):
                    sl = slice(j * P, (j + 1) * P) if offsets == "lane" else slice(0, L)
                    pend[j] = float(v[sl].max())
            rows[t] = total()
        return rows

    A = walk(False)
    Bt = walk(True)
    logz2 = A[T - 1, L - 1]
    g = np.exp2(A + Bt - z[:, y].astype(np.float64) - logz2)
    g /= g.sum(1, keepdims=True)  # the grad kernel normalises every frame by its total
    logz = logz2 / LOG2E + (T - 1) * tmax + float(m.sum())
    return g, logz


def fac_posteriors_float64(e, y, tr):
    """float64 reference of the same posteriors"""
    T, N = e.shape
    L = len(y)
    e = e.astype(np.float64)
    tr = tr.astype(np.float64)
    s1 = tr[y, y]
    s2 = np.full(L, -np.inf)
    s2[1:] = tr[y[1:], y[:-1]]
    A = np.full((T, L), -np.inf)
    Bt = np.full((T, L), -np.inf)
    A[0, 0] = e[0, y[0]]
    for t in range(1, T):
        nb = np.concatenate(([-np.inf], A[t - 1, :-1]))
        A[t] = e[t, y] + np.logaddexp(A[t - 1] + s1, nb + s2)
    Bt[T - 1, L - 1] = e[T - 1, y[L - 1]]
    s2b = np.full(L, -np.inf)
    s2b[:-1] = s2[1:]
    for t in range(T - 2, -1, -1):
        nb = np.concatenate((Bt[t + 1, 1:], [-np.inf]))
        Bt[t] = e[t, y] + np.logaddexp(Bt[t + 1] + s1, nb + s2b)
    g = np.exp(A + Bt - e[:, y] - A[T - 1, L - 1])
    return g / g.sum(1, keepdims=True), A[T - 1, L - 1]


def ctc_chain_emulate(e, y, P=4, kRc=2):
    """float32 arithmetic of the round-2 CTC kernels (criterion_ctc.cu): log-softmax scores of the extended-target labels
    gathered per frame (lp' = (e - lz) * log2e - log2 1.25), three-way log2-sum-exp with lg2(1.25 * sum), P consecutive
    states per lane with one re-centring offset per lane (lagged), alpha and beta stored, posteriors normalised per
    frame.  Returns (loss (natural log, unscaled), d_emis [T][N] = softmax - occupancy)."""
    T, N = e.shape
    L = len(y)
    S = 2 * L + 1
    blank = N - 1
    zlab = np.full(S, blank, np.int64)
    zlab[1::2] = y
    e64 = e.astype(np.float64)
    lz = np.log(np.exp(e64 - e64.max(1, keepdims=True)).sum(1)) + e64.max(1)
    lp = np.maximum(((e64[:, zlab] - lz[:, None]) * LOG2E).astype(F) - LG_SHIFT, NEG).astype(F)  # [T][S], shift folded
    skip_in = np.zeros(S, bool)   # s-2 -> s allowed
    skip_in[3::2] = y[1:] != y[:-1]
    pen_a = np.where(skip_in, F(0), NEG).astype(F)
    pen_b = np.full(S, NEG, F)    # s -> s+2 allowed
    pen_b[:-2] = pen_a[2:]
    nl = (S + P - 1) // P
    lane = np.arange(S) // P

    def lse3(a, b, c):
        mx = np.maximum(np.maximum(a, b), c)
        ssum = (np.exp2((a - mx).astype(F).astype(np.float64)).astype(F) + np.exp2((b - mx).astype(F).astype(np.float64)).astype(F)).astype(F)
        ssum = (ssum + np.exp2((c - mx).astype(F).astype(np.float64)).astype(F)).astype(F)
        return (mx + np.log2((ssum * LG_SCALE).astype(F).astype(np.float64)).astype(F)).astype(F)

    def walk(beta):
        v = np.full(S, NEG, F)
        C = np.zeros(nl, np.float64)
        off = np.zeros(nl)
        pend = np.full(nl, float(NEG))
        rows = np.zeros((T, S), np.float64)
        t0 = T - 1 if beta else 0
        if not beta:
            v[:min(2, S)] = lp[0, :min(2, S)] + LG_SHIFT
        else:
            v[S - 1] = lp[T - 1, S - 1] + LG_SHIFT
            if S > 1:
                v[S - 2] = lp[T - 1, S - 2] + LG_SHIFT
        rows[t0] = v.astype(np.float64) + C[lane]
        for t in (range(T - 2, -1, -1) if beta else range(1, T)):
            Cl = C[lane]
            if not beta:
                n1 = np.concatenate(([NEG], v[:-1]))
                n2 = np.concatenate(([NEG, NEG], v[:-2]))
                d1 = np.concatenate(([0.0], Cl[:-1] - Cl[1:]))
                d2 = np.concatenate(([0.0, 0.0], Cl[:-2] - Cl[2:]))
                pen = pen_a
            else:
                n1 = np.concatenate((v[1:], [NEG]))
                n2 = np.concatenate((v[2:], [NEG, NEG]))
                d1 = np.concatenate((Cl[1:] - Cl[:-1], [0.0]))
                d2 = np.concatenate((Cl[2:] - Cl[:-2], [0.0, 0.0]))
                pen = pen_b
            n1 = (n1 + d1.astype(F)).astype(F)
            n2 = ((n2 + d2.astype(F)).astype(F) + pen).astype(F)
            v = (lp[t] + lse3(v, n1, n2)).astype(F)
            if (t % kRc) == (kRc - 1 if beta else 0):
                for j in range(nl):
                    sl = slice(j * P, (j + 1) * P)
                    if pend[j] > -1e29:
                        off_new = min(max(0.5 * (off[j] - pend[j]), 0.0), 48.0)
                        mm = F(pend[j] - off_new)
                        off[j] = off_new
                        v[sl] = (v[sl] - mm).astype(F)
                        C[j] += float(mm)
                    else:
                        jn = j + 1 if beta else j - 1
                        if 0 <= jn < nl:
                            v[sl] = (v[sl] - F(C[jn] - C[j])).astype(F)
                            C[j] = C[jn]
            if (t % kRc) == (0 if beta else kRc - 1):
                for j in range(nl):
                    pend[j] = float(v[j * P:(j + 1) * P].max())
            rows[t] = v.astype(np.float64) + C[lane]
        return rows

    A = walk(False)
    Bt = walk(True)
    last = [A[T - 1, S - 1]] + ([A[T - 1, S - 2]] if S > 1 else [])
    ll2 = max(last) + np.log2(sum(2.0 ** (x - max(last)) for x in last))
    lp_true = lp.astype(np.float64) + float(LG_SHIFT)
    post = np.exp2(A + Bt - lp_true - ll2)
    post /= post.sum(1, keepdims=True)
    occ = np.zeros((T, N))
    for s_ in range(S):
        occ[:, zlab[s_]] += post[:, s_]
    soft = np.exp(e64 - lz[:, None])
    return -ll2 / LOG2E, soft - occ


def layernorm_rows_emulate(x, V, pivot="sample", eps=1e-5):
    """float32 arithmetic of the statistics of ln_row_fwd_kernel<V> (am_kernels.cu): one warp per group, lane l sums the
    V-wide chunks at V*l, V*l + 32V, ... in fp32 (V = 4 folds a chunk as (x + y) + (z + w) and its squares as
    fma(y, y, x*x) + fma(w, w, z*z)), the lanes' sums are combined in double.  The sums are taken about a pivot K:
    "sample" (the kernel's: plain sums, and where they cancel (mean^2 > 64 var) sums again about the mean of the values at
    l * R / 32, l = 0..31, added by a warp's xor butterfly), "first" (the first value) or "none" (K = 0, the one-pass
    Q/R - mean^2).  x [G][R] float32 -> xhat = (x - mu) * rstd [G][R], mu [G], rstd [G], float32."""
    G, R = x.shape
    x = x.astype(F)

    def fma(a, b, c):
        return (a.astype(np.float64) * b + c).astype(F)

    def sums(K):
        s, q = np.zeros((G, 32), F), np.zeros((G, 32), F)
        for i0 in range(0, R, V):
            lane = (i0 // V) % 32
            d = (x[:, i0:i0 + V] - K[:, None]).astype(F)
            if V == 4:
                cs = (d[:, 0] + d[:, 1]) + (d[:, 2] + d[:, 3])
                cq = fma(d[:, 1], d[:, 1], d[:, 0] * d[:, 0]) + fma(d[:, 3], d[:, 3], d[:, 2] * d[:, 2])
            else:
                cs, cq = d[:, 0], d[:, 0] * d[:, 0]
            s[:, lane] += cs
            q[:, lane] += cq
        return s.astype(np.float64).sum(1) / R, q.astype(np.float64).sum(1) / R

    K = x[:, 0].copy() if pivot == "first" else np.zeros(G, F)
    S, Q = sums(K)
    if pivot == "sample":
        v = x[:, np.arange(32) * R // 32]
        for o in (16, 8, 4, 2, 1):  # the xor butterfly of warp_sum
            v = v + v[:, np.arange(32) ^ o]
        cancels = S * S > 64 * (Q - S * S)
        K = np.where(cancels, v[:, 0] * F(1 / 32), F(0)).astype(F)
        S2, Q2 = sums(K)
        S, Q = np.where(cancels, S2, S), np.where(cancels, Q2, Q)
    mu = (K.astype(np.float64) + S).astype(F)
    rstd = (1.0 / np.sqrt(np.maximum(Q - S * S, 0.0) + float(F(eps)))).astype(F)
    return ((x - mu[:, None]) * rstd[:, None]).astype(F), mu, rstd
