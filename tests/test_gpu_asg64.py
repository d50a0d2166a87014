"""The 64-wide ASG and FCC-Viterbi entry points (w2l_asg64_forward_backward, w2l_fcc_viterbi64) for
1 <= N <= 64 against the CPU oracle, with the tolerances of test_gpu_criterion.py: loss and gradients
<= 1e-4 relative, Viterbi paths bit-exact."""
import functools

import numpy as np
import pytest

import oracle
from test_gpu_criterion import TOL, check_asg, dev, make_asg, rel

pytestmark = pytest.mark.gpu

check_asg64 = functools.partial(check_asg, entry="asg64_forward_backward")


@pytest.mark.parametrize("B,T,N,L,mode", [
    (1, 1, 33, 1, "none"), (2, 2, 39, 2, "none"), (3, 3, 64, 3, "input_sz"), (3, 17, 61, 5, "target_sz"),
    (4, 100, 39, 20, "target_sz_sqrt"), (2, 101, 64, 33, "input_sz_sqrt"), (5, 64, 1, 7, "none"),
    (4, 300, 48, 60, "target_sz_sqrt"), (3, 40, 5, 100, "none"), (2, 257, 39, 257, "none"),
    (2, 500, 32, 90, "input_sz"), (2, 1500, 61, 300, "target_sz_sqrt"),
    (3, 700, 39, 666, "target_sz_sqrt"), (2, 1100, 64, 1000, "none"),  # long targets: the sliced (halo) FAC gradient path
])
def test_asg64_parity(B, T, N, L, mode):
    e, tr, y = make_asg(B, T, N, L, seed=B * 1000 + T + N)
    check_asg64(e, tr, y, mode)


def test_asg64_dloss_and_terms():
    import wav2letter_b200 as w

    e, tr, y = make_asg(4, 120, 39, 25, seed=11)
    g = np.random.default_rng(3).normal(0, 1, 4).astype(np.float32)
    check_asg64(e, tr, y, "target_sz", dloss=g)
    check_asg64(e, tr, y, "none", terms=w.TERM_FCC)
    check_asg64(e, tr, y, "target_sz", terms=w.TERM_FAC)


def test_asg64_invalid_targets_give_nan_loss_and_zero_grad():
    import wav2letter_b200 as w

    e, tr, y = make_asg(3, 30, 39, 6, seed=13, ragged=False)
    y[0, :] = -1
    y[2, 1] = 39  # one past the last token
    gl, gde, gdt = w.asg64_forward_backward(dev(e), dev(y), dev(tr))
    gl, gde = gl.cpu().numpy(), gde.cpu().numpy()
    assert np.isnan(gl[0]) and np.isnan(gl[2]) and np.isfinite(gl[1])
    assert not gde[0].any() and not gde[2].any() and gde[1].any()
    ol, ode, odt = oracle.asg(e, y, tr)
    assert rel(gde, ode) <= TOL and rel(gdt.cpu().numpy(), odt) <= TOL


def test_asg64_baseline_size_and_zero_sum_property():
    """B = 64, T = 1500 at N = 61: oracle parity, per-frame gradient sums vanish, and a second run is bit-identical."""
    import wav2letter_b200 as w

    B, T, N, L = 64, 1500, 61, 250
    e, tr, y = make_asg(B, T, N, L, seed=7)
    gl, gde, gdt = check_asg64(e, tr, y, "target_sz_sqrt")
    assert np.abs(gde.sum(axis=2)).max() < 1e-4  # gamma_fcc and gamma_fac both sum to 1 per frame
    assert abs(gdt.sum()) < 2e-2 * np.abs(gdt).sum() / gdt.size + 1e-2
    gl2, gde2, gdt2 = (x.cpu().numpy() for x in w.asg64_forward_backward(dev(e), dev(y), dev(tr), "target_sz_sqrt"))
    assert np.array_equal(gl, gl2) and np.array_equal(gde, gde2) and np.array_equal(gdt, gdt2)


@pytest.mark.parametrize("N", [1, 5, 30, 32])
def test_asg64_agrees_with_the_32_wide_call(N):
    """Both calls evaluate the same recursions in fp32; the 64-wide FCC chains sum the matrix-vector product in another
    order, so the results agree to rounding, not bit for bit."""
    import wav2letter_b200 as w

    e, tr, y = make_asg(4, 400, N, 60, seed=N)
    a = [x.cpu().numpy() for x in w.asg_forward_backward(dev(e), dev(y), dev(tr), "target_sz_sqrt")]
    b = [x.cpu().numpy() for x in w.asg64_forward_backward(dev(e), dev(y), dev(tr), "target_sz_sqrt")]
    assert np.abs(a[0] - b[0]).max() <= 1e-5 * max(1.0, np.abs(a[0]).max())
    assert rel(b[1], a[1]) <= 1e-5
    assert rel(b[2], a[2], 1e-2 * 4 * 400 if N == 1 else 2e-3) <= 1e-5


@pytest.mark.parametrize("B,T,N", [(1, 1, 33), (3, 2, 39), (4, 333, 61), (8, 1500, 64), (2, 4000, 39), (1, 7000, 61)])
def test_fcc_viterbi64_bit_exact(B, T, N):
    import wav2letter_b200 as w

    e, tr, _ = make_asg(B, T, N, 1, seed=T + N)
    p = w.fcc_viterbi64(dev(e), dev(tr)).cpu().numpy()
    np.testing.assert_array_equal(p, oracle.fcc_viterbi(e, tr))
    p2 = w.fcc_viterbi64(dev(e), dev(tr)).cpu().numpy()
    np.testing.assert_array_equal(p, p2)


@pytest.mark.parametrize("N", [33, 64])
def test_fcc_viterbi64_ties(N):
    import wav2letter_b200 as w

    e = np.zeros((3, 9, N), np.float32)
    tr = np.zeros((N, N), np.float32)
    e[1, 4, N - 1] = 1.0
    e[2, :, 31] = e[2, :, 32] = 1.0  # tied states 31 (lane 31) and 32 (lane 0's second state): the first one wins
    p = w.fcc_viterbi64(dev(e), dev(tr)).cpu().numpy()
    np.testing.assert_array_equal(p, oracle.fcc_viterbi(e, tr))
    assert p[0].tolist() == [0] * 9 and p[2].tolist() == [31] * 9


@pytest.mark.parametrize("B,T,N", [(2, 50, 1), (4, 333, 30), (2, 4000, 32)])
def test_fcc_viterbi64_equals_the_32_wide_call(B, T, N):
    import wav2letter_b200 as w

    e, tr, _ = make_asg(B, T, N, 1, seed=T)
    np.testing.assert_array_equal(w.fcc_viterbi64(dev(e), dev(tr)).cpu().numpy(), w.fcc_viterbi(dev(e), dev(tr)).cpu().numpy())


def test_n65_is_unsupported():
    import wav2letter_b200 as w

    e = np.zeros((1, 5, 65), np.float32)
    tr = np.zeros((65, 65), np.float32)
    with pytest.raises(w.W2LError) as ei:
        w.asg64_forward_backward(dev(e), dev(np.zeros((1, 2), np.int32)), dev(tr))
    assert ei.value.code == 4
    with pytest.raises(w.W2LError) as ei:
        w.fcc_viterbi64(dev(e), dev(tr))
    assert ei.value.code == 4
