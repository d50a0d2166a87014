"""CPU check of the arithmetic formulation used by the CUDA ASG, CTC and per-row LayerNorm kernels (see
tests/kernel_math_emulation.py) against the oracle, incl. adversarial emission ranges."""
import numpy as np
import pytest

import oracle
from kernel_math_emulation import (ctc_chain_emulate, fac_chain_emulate, fac_emulate, fac_posteriors_float64, fcc_emulate,
                                   layernorm_rows_emulate)


def rel(a, b):
    return float(np.abs(a - b).max() / max(1e-30, np.abs(b).max()))


@pytest.mark.parametrize("T,N,scale,seed", [(1, 5, 3, 0), (2, 30, 3, 1), (50, 30, 3, 2), (400, 30, 3, 3),
                                            (300, 30, 60, 4), (257, 7, 10, 5)])
def test_fcc_linear_domain_formulation(T, N, scale, seed):
    rng = np.random.default_rng(seed)
    e = (rng.normal(0, 1, (T, N)) * scale).astype(np.float32)
    tr = (4 * np.eye(N) + rng.normal(0, 0.1, (N, N))).astype(np.float32)
    logz, gamma, xi = fcc_emulate(e, tr)
    l, de, dtr = oracle.fcc(e[None], tr)
    assert abs(logz - l[0]) <= 2e-6 * abs(l[0]) + 1e-5
    assert rel(gamma, de[0]) < 2e-5
    if T > 1:
        assert rel(xi, dtr) < 2e-5


@pytest.mark.parametrize("T,N,L,scale,seed", [(1, 4, 1, 3, 0), (2, 5, 2, 3, 1), (3, 5, 1, 3, 2), (40, 30, 9, 3, 3),
                                              (301, 30, 60, 3, 4), (200, 30, 200, 3, 5), (300, 30, 50, 60, 6)])
def test_fac_meet_in_the_middle_formulation(T, N, L, scale, seed):
    rng = np.random.default_rng(50 + seed)
    e = (rng.normal(0, 1, (T, N)) * scale).astype(np.float32)
    tr = (4 * np.eye(N) + rng.normal(0, 0.1, (N, N))).astype(np.float32)
    y = rng.integers(0, N, L).astype(np.int32)
    logz, G, dtr = fac_emulate(e, y, tr)
    l, de, dt = oracle.fac(e[None], y[None], tr)
    assert abs(logz - l[0]) <= 2e-6 * abs(l[0]) + 1e-5
    tol = 1e-4 if scale <= 3 else 2e-3  # x20 emissions: fp32 log-domain rounding, see DESIGN.md
    assert rel(G, de[0]) < tol
    if T > 1:
        assert rel(dtr, dt) < tol


@pytest.mark.parametrize("scale", [3, 60])
def test_fcc_rescale_controller_is_stable(scale):
    """The alpha walk's lag-two rescale must be damped: undamped it leaves fp32 range (this bug
    was seen on the GPU as NaN transition gradients at T=1500)."""
    worst_damped, worst_undamped = 0.0, 0.0
    for seed in range(6):
        rng = np.random.default_rng(900 + seed)
        e = (rng.normal(0, 1, (1500, 30)) * scale).astype(np.float32)
        tr = (4 * np.eye(30) + rng.normal(0, 0.1, (30, 30))).astype(np.float32)
        worst_damped = max(worst_damped, float(np.abs(fcc_emulate(e, tr, 1, True)).max()))
        ex = fcc_emulate(e, tr, 0, True)
        worst_undamped = max(worst_undamped, float(np.abs(ex[np.isfinite(ex)]).max()))
    assert worst_damped < 40
    if scale == 3:
        assert worst_undamped > 60  # documents why the damping is there


@pytest.mark.parametrize("T,N,L,scale,seed", [(1, 4, 1, 3, 0), (2, 5, 2, 3, 1), (40, 30, 9, 3, 3), (301, 30, 60, 3, 4), (200, 30, 200, 3, 5)])
def test_fac_round2_chain_formulation(T, N, L, scale, seed):
    """the log2-domain recursion of the round-2 kernels (per-lane offsets, lagged re-centring, lg2(1.25 (1+r)) with the
    shift folded into the transition scores) against float64"""
    rng = np.random.default_rng(70 + seed)
    e = (rng.normal(0, 1, (T, N)) * scale).astype(np.float32)
    tr = (4 * np.eye(N) + rng.normal(0, 0.1, (N, N))).astype(np.float32)
    y = rng.integers(0, N, L).astype(np.int32)
    g, logz = fac_chain_emulate(e, y, tr, "lane")
    g64, logz64 = fac_posteriors_float64(e, y, tr)
    assert abs(logz - logz64) <= 1e-5 * abs(logz64) + 1e-5  # fp32 accumulation over T steps (north star: 1e-4 relative)
    assert np.abs(g - g64).max() < 2e-5


def test_fac_per_lane_offsets_keep_tight_bands_accurate():
    """Why the chains keep one re-centring offset per lane: with one offset per row the states far below the row maximum
    — which carry the posterior mass when the alignment band is tight (L close to T) — lose absolute precision.
    (Measured on the GPU: 2.9e-4 -> within 1e-4 on T = 700, L = 540; 7e-4 -> 8e-5 at T = 4000.)"""
    rng = np.random.default_rng(3 * 1000 + 700)
    T, N, L = 400, 30, 330
    e = (rng.normal(0, 1, (T, N)) * 3).astype(np.float32)
    tr = (4 * np.eye(N) + rng.normal(0, 0.1, (N, N))).astype(np.float32)
    y = rng.integers(0, N, L).astype(np.int32)
    g64, _ = fac_posteriors_float64(e, y, tr)
    err_lane = np.abs(fac_chain_emulate(e, y, tr, "lane")[0] - g64).max()
    err_row = np.abs(fac_chain_emulate(e, y, tr, "row")[0] - g64).max()
    assert err_lane < 2e-5
    assert err_row > 3 * err_lane  # documents why the offsets are per lane


@pytest.mark.parametrize("T,N,L,seed", [(1, 5, 0, 0), (3, 6, 1, 1), (30, 12, 9, 2), (150, 200, 60, 3), (90, 40, 44, 4)])
def test_ctc_round2_chain_formulation(T, N, L, seed):
    """the log2-domain three-way recursion of the round-2 CTC kernels (per-lane offsets, lagged re-centring, lg2(1.25 x))
    against the oracle, repeated labels and a tight band (2L+1 close to T) included"""
    rng = np.random.default_rng(90 + seed)
    e = (rng.normal(0, 1, (T, N)) * 3).astype(np.float32)
    y = rng.integers(0, N - 1, L).astype(np.int32)
    if L > 4:
        y[3] = y[2]  # an adjacent repeat: no skip transition there
    if T < 2 * L + 1 - L:  # keep the target feasible
        return
    loss, grad = ctc_chain_emulate(e, y)
    ol, og = oracle.ctc(e[None], y[None] if L else np.full((1, 1), -1, np.int32), "none")
    assert abs(loss - ol[0]) <= 1e-5 * abs(ol[0]) + 1e-5
    assert rel(grad, og[0]) < 2e-5


def test_halo_slices_reproduce_the_full_row():
    """The sliced FAC gradient path (asg_fac_grad_halo_kernel): within an 8-frame segment the recursion reaches only 8
    positions sideways, so a slice of 240 useful positions with an 8-position halo on either side, started from the full
    row's checkpoint and cut off from its neighbours, reproduces the full row on its useful positions exactly."""
    rng = np.random.default_rng(11)
    L, N, steps = 700, 30, 8
    y = rng.integers(0, N, L)
    tr = 4 * np.eye(N) + rng.normal(0, 0.1, (N, N))
    s1 = tr[y, y]
    s2a = np.full(L, -np.inf)
    s2a[1:] = tr[y[1:], y[:-1]]
    s2b = np.full(L, -np.inf)
    s2b[:-1] = s2a[1:]
    e = rng.normal(0, 3, (steps, N))

    def alpha_steps(row, sa1, sa2, lab):
        for t in range(steps):
            nb = np.concatenate(([-np.inf], row[:-1]))
            row = e[t, lab] + np.logaddexp(row + sa1, nb + sa2)
        return row

    def beta_steps(row, sb1, sb2, lab):
        for t in range(steps - 1, -1, -1):
            nb = np.concatenate((row[1:], [-np.inf]))
            row = e[t, lab] + np.logaddexp(row + sb1, nb + sb2)
        return row

    a0 = rng.normal(-20, 10, L)
    b0 = rng.normal(-20, 10, L)
    full_a, full_b = alpha_steps(a0, s1, s2a, y), beta_steps(b0, s1, s2b, y)
    for w in range((L + 239) // 240):
        base = 240 * w - 8
        idx = np.arange(base, base + 256)
        ok = (idx >= 0) & (idx < L)
        ii = np.clip(idx, 0, L - 1)
        pick = lambda x, dead: np.where(ok, x[ii], dead)  # noqa: E731
        lab = np.where(ok, y[ii], 0)
        sl_a = alpha_steps(pick(a0, -np.inf), pick(s1, 0.0), pick(s2a, -np.inf), lab)
        sl_b = beta_steps(pick(b0, -np.inf), pick(s1, 0.0), pick(s2b, -np.inf), lab)
        use = ok & (np.arange(256) >= 8) & (np.arange(256) < 248)
        np.testing.assert_array_equal(sl_a[use], full_a[idx[use]])
        np.testing.assert_array_equal(sl_b[use], full_b[idx[use]])


def _xhat_err(x, xhat, eps=1e-5):
    x64 = x.astype(np.float64)
    m = x64.mean(1, keepdims=True)
    ref = (x64 - m) / np.sqrt(((x64 - m) ** 2).mean(1, keepdims=True) + eps)
    return rel(xhat, ref)


@pytest.mark.parametrize("V", [4, 1])
def test_layernorm_row_sums_about_a_pivot(V):
    """Why the per-row LayerNorm sums about a pivot: its fp32 lane sums lose about 2 log10(mean / sigma) digits in
    Q/R - mean^2 (1e-2 of the output at mean / sigma = 1e3, the variance clamped to 0 at 1e4), and about the mean of
    32 values spread over the group (used where the plain sums cancel: mean above 8 sigma) they lose none: what remains is
    the fp32 rounding of the stored mean (half an ulp of 1e4 is 5e-4 sigma).  The pivot is a mean because a first value
    50 sigma off the mean would cost 2 log10(50) digits; well-conditioned rows (post-ReLU: half of them zeros) keep the
    plain sums."""
    rng = np.random.default_rng(40 + V)
    G, R = 64, 640
    bound = {0.5: 3e-7, 30: 1e-6, 1e3: 3e-5, 1e4: 5e-4}
    for ratio, tol in bound.items():
        x = rng.normal(ratio, 1.0, (G, R)).astype(np.float32)
        assert _xhat_err(x, layernorm_rows_emulate(x, V)[0]) < tol, ratio
        if ratio >= 1e3:
            assert _xhat_err(x, layernorm_rows_emulate(x, V, "none")[0]) > 100 * tol, ratio  # the unshifted sums
    x = rng.normal(0.0, 1.0, (G, R)).astype(np.float32)
    x[:, 0] = 50.0
    assert _xhat_err(x, layernorm_rows_emulate(x, V)[0]) < 3e-7
    assert _xhat_err(x, layernorm_rows_emulate(x, V, "first")[0]) > 3e-6  # the first value as the pivot
    x = (np.maximum(rng.normal(0.0, 1.0, (256, 2160)), 0) * 1.3).astype(np.float32)
    assert _xhat_err(x, layernorm_rows_emulate(x, V)[0]) < 5e-7
    for c in (17.7, 3.3, -250.1, 0.0):  # a constant group, also shorter than the 32 samples: exact mean, variance 0, xhat 0
        for n in (4, 12, 1200):
            xhat, mu, rstd = layernorm_rows_emulate(np.full((2, n), c, np.float32), V)
            assert (xhat == 0).all() and (mu == np.float32(c)).all()
            assert (rstd == np.float32(1 / np.sqrt(float(np.float32(1e-5))))).all()
