"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded
inputs, against the committed golden fixtures, and through size-independent properties at the
BASELINE sizes.  Tolerances: loss and gradients <= 1e-4 relative (north_star), Viterbi paths
bit-exact."""
import os

import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-4


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rel(a, b, floor=2e-3):
    """max abs error over max abs reference; `floor` = scale of the cancelling components when the
    reference itself is ~0 (N = 1: gamma_fcc - gamma_fac = 1 - 1, d_trans = (T-1) - (T-1))."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(floor, np.abs(b).max()))


def make_asg(B, T, N, L, seed, escale=3.0, ragged=True):
    rng = np.random.default_rng(seed)
    e = (rng.normal(0, 1, (B, T, N)) * escale).astype(np.float32)
    tr = (4 * np.eye(N) + rng.normal(0, 0.1, (N, N))).astype(np.float32)
    y = rng.integers(0, N, (B, L)).astype(np.int32)
    if ragged and L > 1:
        for b in range(B):
            n = int(rng.integers(max(1, L // 2), L + 1))
            y[b, n:] = -1
    return e, tr, y


def check_asg(e, tr, y, mode="none", dloss=None, terms=None, tol=TOL, entry="asg_forward_backward"):
    """`entry`: the wav2letter_b200 call under test (asg_forward_backward or asg64_forward_backward)."""
    import wav2letter_b200 as w

    fb = getattr(w, entry)
    terms = w.TERM_ASG if terms is None else terms
    fn = {w.TERM_ASG: oracle.asg, w.TERM_FAC: oracle.fac}.get(terms)
    if terms == w.TERM_FCC:
        ol, ode, odt = oracle.fcc(e, tr, mode, target=y, dloss=dloss)
    else:
        ol, ode, odt = fn(e, y, tr, mode, dloss=dloss)
    gl, gde, gdt = fb(dev(e), dev(y), dev(tr), mode, None if dloss is None else dev(dloss), terms)
    torch.cuda.synchronize()
    gl, gde, gdt = gl.cpu().numpy(), gde.cpu().numpy(), gdt.cpu().numpy()
    lerr = np.abs(gl - ol) / np.maximum(1.0, np.abs(ol))
    assert np.nanmax(lerr) <= tol, f"loss rel err {np.nanmax(lerr)}"
    assert np.array_equal(np.isnan(gl), np.isnan(ol))
    assert rel(gde, ode) <= tol, f"d_emis rel err {rel(gde, ode)}"
    if e.shape[1] > 1:
        floor = 1e-2 * e.shape[0] * e.shape[1]  # each of FCC / FAC contributes ~B*(T-1) mass
        assert rel(gdt, odt, floor if e.shape[2] == 1 else 2e-3) <= tol, f"d_trans rel err {rel(gdt, odt)}"
    # forward-only entry gives the same loss
    fl, _, _ = fb(dev(e), dev(y), dev(tr), mode, None, terms, need_grad=False)
    np.testing.assert_allclose(fl.cpu().numpy(), ol, rtol=tol, atol=tol)
    return gl, gde, gdt


@pytest.mark.parametrize("B,T,N,L,mode", [
    (1, 1, 5, 1, "none"), (2, 2, 3, 2, "none"), (3, 3, 4, 3, "input_sz"), (3, 17, 30, 5, "target_sz"),
    (4, 100, 30, 20, "target_sz_sqrt"), (2, 101, 32, 33, "input_sz_sqrt"), (5, 64, 1, 7, "none"),
    (8, 500, 30, 80, "target_sz_sqrt"), (2, 257, 30, 257, "none"), (3, 40, 30, 100, "none"),
    (3, 700, 30, 666, "target_sz_sqrt"), (2, 1100, 28, 1000, "none"),  # long targets: the sliced (halo) FAC gradient path
])
def test_asg_parity(B, T, N, L, mode):
    e, tr, y = make_asg(B, T, N, L, seed=B * 1000 + T)
    check_asg(e, tr, y, mode)


def test_asg_parity_baseline_size_and_zero_sum_property():
    """T=1500, N=30, B=64 (BASELINE.json): oracle parity + per-frame gradient sums vanish."""
    B, T, N, L = 64, 1500, 30, 250
    e, tr, y = make_asg(B, T, N, L, seed=7)
    gl, gde, gdt = check_asg(e, tr, y, "target_sz_sqrt")
    assert np.abs(gde.sum(axis=2)).max() < 1e-4  # gamma_fcc and gamma_fac both sum to 1 per frame
    assert abs(gdt.sum()) < 2e-2 * np.abs(gdt).sum() / gdt.size + 1e-2


def test_asg_dloss_terms_and_adversarial():
    import wav2letter_b200 as w

    e, tr, y = make_asg(4, 120, 30, 25, seed=11)
    g = np.random.default_rng(3).normal(0, 1, 4).astype(np.float32)
    check_asg(e, tr, y, "target_sz", dloss=g)
    check_asg(e, tr, y, "none", terms=w.TERM_FCC)
    check_asg(e, tr, y, "target_sz", terms=w.TERM_FAC)
    e2, tr2, y2 = make_asg(3, 300, 30, 50, seed=12, escale=60.0)  # emissions x20: one-hot-ish posteriors
    check_asg(e2, tr2, y2, "none", tol=2e-3)


def test_asg_invalid_targets_give_nan_loss_and_zero_grad():
    import wav2letter_b200 as w

    e, tr, y = make_asg(3, 30, 30, 6, seed=13, ragged=False)
    y[0, :] = -1
    y[2, 1] = 99
    gl, gde, gdt = w.asg_forward_backward(dev(e), dev(y), dev(tr))
    gl, gde = gl.cpu().numpy(), gde.cpu().numpy()
    assert np.isnan(gl[0]) and np.isnan(gl[2]) and np.isfinite(gl[1])
    assert not gde[0].any() and not gde[2].any() and gde[1].any()
    ol, ode, odt = oracle.asg(e, y, tr)
    assert rel(gde, ode) <= TOL and rel(gdt.cpu().numpy(), odt) <= TOL


def test_linseg_is_fac_on_stretched_target():
    import wav2letter_b200 as w

    e, tr, y = make_asg(3, 50, 30, 9, seed=14)
    st = w.linseg_target(dev(y), 50)
    np.testing.assert_array_equal(st.cpu().numpy(), oracle.linseg_target(y, 50))
    check_asg(e, tr, st.cpu().numpy(), "none", terms=w.TERM_FAC)


@pytest.mark.parametrize("B,T,N", [(1, 1, 4), (3, 2, 30), (4, 333, 30), (64, 1500, 30), (2, 4000, 32), (1, 7000, 30)])
def test_fcc_viterbi_bit_exact(B, T, N):
    import wav2letter_b200 as w

    e, tr, _ = make_asg(B, T, N, 1, seed=T)
    p = w.fcc_viterbi(dev(e), dev(tr)).cpu().numpy()
    np.testing.assert_array_equal(p, oracle.fcc_viterbi(e, tr))


def test_fcc_viterbi_ties_and_path_optimality():
    import wav2letter_b200 as w

    e = np.zeros((2, 9, 6), np.float32)
    tr = np.zeros((6, 6), np.float32)
    e[1, 4, 5] = 1.0
    p = w.fcc_viterbi(dev(e), dev(tr)).cpu().numpy()
    np.testing.assert_array_equal(p, oracle.fcc_viterbi(e, tr))
    assert p[0].tolist() == [0] * 9
    # property at full size: the Viterbi path beats random paths and FCC >= its score
    B, T, N = 8, 1500, 30
    e, tr, _ = make_asg(B, T, N, 1, seed=5)
    p = w.fcc_viterbi(dev(e), dev(tr)).cpu().numpy()

    def score(path, b):
        return e[b, np.arange(T), path].astype(np.float64).sum() + tr[path[1:], path[:-1]].astype(np.float64).sum()

    fcc = oracle.fcc(e, tr, backward=False)
    rng = np.random.default_rng(0)
    for b in range(B):
        s = score(p[b], b)
        assert fcc[b] >= s - 1e-3
        for _ in range(5):
            q = p[b].copy()
            k = rng.integers(0, T, 20)
            q[k] = rng.integers(0, N, 20)
            assert score(q, b) <= s + 1e-3


@pytest.mark.parametrize("B,T,N,L", [(1, 1, 4, 1), (3, 7, 5, 7), (4, 200, 30, 40), (16, 1500, 30, 250), (2, 3000, 30, 900)])
def test_fac_viterbi_bit_exact(B, T, N, L):
    import wav2letter_b200 as w

    e, tr, y = make_asg(B, T, N, L, seed=T + L)
    p, idx = w.fac_viterbi(dev(e), dev(y), dev(tr), return_index=True)
    op, oidx = oracle.fac_viterbi(e, y, tr, return_index=True)
    np.testing.assert_array_equal(idx.cpu().numpy(), oidx)
    np.testing.assert_array_equal(p.cpu().numpy(), op)


def make_ctc(B, T, N, L, seed, escale=2.0):
    rng = np.random.default_rng(seed)
    e = (rng.normal(0, 1, (B, T, N)) * escale).astype(np.float32)
    y = rng.integers(0, N - 1, (B, max(L, 1))).astype(np.int32)
    if L == 0:
        y[:] = -1
    for b in range(B):
        if L > 2 and b % 2 == 1:
            n = int(rng.integers(1, L + 1))
            y[b, n:] = -1
        if L > 3 and b % 3 == 0:
            y[b, 1:3] = y[b, 0]
    return e, y


@pytest.mark.parametrize("B,T,N,L,mode", [
    (1, 1, 3, 1, "none"), (2, 5, 6, 2, "none"), (3, 12, 5, 12, "target_sz"), (4, 150, 31, 40, "target_sz"),
    (8, 400, 31, 120, "input_sz"), (2, 60, 1000, 20, "none"), (2, 40, 9998, 12, "target_sz_sqrt"), (2, 30, 31, 0, "none"),
    (2, 700, 31, 600, "none"),
])
def test_ctc_parity(B, T, N, L, mode):
    import wav2letter_b200 as w

    e, y = make_ctc(B, T, N, L, seed=T * 7 + N)
    g = np.random.default_rng(1).uniform(0.5, 2.0, B).astype(np.float32)
    ol, ode = oracle.ctc(e, y, mode, dloss=g)
    gl, gde = w.ctc_forward_backward(dev(e), dev(y), mode, dev(g))
    torch.cuda.synchronize()
    gl, gde = gl.cpu().numpy(), gde.cpu().numpy()
    assert np.max(np.abs(gl - ol) / np.maximum(1, np.abs(ol))) <= TOL
    assert rel(gde, ode) <= TOL, rel(gde, ode)
    assert np.abs(gde.sum(axis=2)).max() < 1e-4 * max(1.0, float(g.max()))  # softmax - occupancy sums to 0
    fl, _ = w.ctc_forward_backward(dev(e), dev(y), mode, None, need_grad=False)
    np.testing.assert_allclose(fl.cpu().numpy(), ol, rtol=TOL, atol=TOL)


def test_ctc_tensorflow_vectors_on_gpu():
    import wav2letter_b200 as w
    from test_oracle_pins import TF_P0, TF_P1

    l0, _ = w.ctc_forward_backward(dev(np.log(np.asarray(TF_P0, np.float32))[None]), dev(np.array([[0, 1, 2, 1, 0]], np.int32)))
    l1, _ = w.ctc_forward_backward(dev(np.log(np.asarray(TF_P1, np.float32))[None]), dev(np.array([[0, 1, 1, 0]], np.int32)))
    assert abs(l0.item() - 3.34211) < 1e-4 and abs(l1.item() - 5.42262) < 1e-4


def test_argmax_path():
    import wav2letter_b200 as w

    e, _ = make_ctc(3, 50, 77, 3, seed=9)
    e[0, 3, :] = 0.5  # all tied -> first index
    np.testing.assert_array_equal(w.argmax_path(dev(e)).cpu().numpy(), oracle.argmax_path(e))


def test_golden_fixtures():
    import wav2letter_b200 as w

    g = np.load(os.path.join(ROOT, "tests", "golden", "criterion_goldens.npz"))
    gl, gde, gdt = w.asg_forward_backward(dev(g["asg_emis"]), dev(g["asg_target"]), dev(g["asg_trans"]), "target_sz_sqrt")
    assert np.max(np.abs(gl.cpu().numpy() - g["asg_loss"]) / np.maximum(1, np.abs(g["asg_loss"]))) <= TOL
    assert rel(gde.cpu().numpy(), g["asg_d_emis"]) <= TOL
    assert rel(gdt.cpu().numpy(), g["asg_d_trans"]) <= TOL
    np.testing.assert_array_equal(w.fcc_viterbi(dev(g["asg_emis"]), dev(g["asg_trans"])).cpu().numpy(), g["asg_viterbi"])
    p, idx = w.fac_viterbi(dev(g["asg_emis"]), dev(g["asg_target"]), dev(g["asg_trans"]), return_index=True)
    np.testing.assert_array_equal(p.cpu().numpy(), g["fac_viterbi"])
    np.testing.assert_array_equal(idx.cpu().numpy(), g["fac_viterbi_idx"])
    cl, cde = w.ctc_forward_backward(dev(g["ctc_emis"]), dev(g["ctc_target"]), "target_sz")
    assert np.max(np.abs(cl.cpu().numpy() - g["ctc_loss"]) / np.maximum(1, np.abs(g["ctc_loss"]))) <= TOL
    assert rel(cde.cpu().numpy(), g["ctc_d_emis"]) <= TOL


def test_error_codes_on_device():
    import wav2letter_b200 as w

    e, tr, y = make_asg(2, 10, 30, 4, seed=1)
    with pytest.raises(w.W2LError) as ei:
        w.asg_forward_backward(dev(e), dev(y), dev(tr), ws=torch.empty(16, dtype=torch.uint8, device="cuda"))
    assert ei.value.code == 2
    e40 = np.zeros((1, 5, 40), np.float32)
    with pytest.raises(w.W2LError) as ei:
        w.asg_forward_backward(dev(e40), dev(np.zeros((1, 2), np.int32)), dev(np.zeros((40, 40), np.float32)))
    assert ei.value.code == 4
