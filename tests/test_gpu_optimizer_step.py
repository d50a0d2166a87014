"""The optimizer end of a training step against a float64 model of Train.cpp's rule (:1743-1803):

    s = 1 / total_batch
    n = sqrt(sum G^2 + [clampCrit] sum Gc^2)          clampCrit: ctc / asg yes, the linseg warm start no (:1878,1923,1939)
    c = M / (n s + 1e-6) if M > 0 and n s > M else 1  (fl::clipGradNorm over the scaled gradients)
    v <- mu v + G s c ;  p <- p - lr v                (network: SGD with momentum)
    t <- t - lrcrit Gc s [clampCrit ? c : 1]          (criterion: plain SGD, never momentum)

and a device-side guard that skips the whole update when the loss or a gradient norm is not finite.

Every step is checked from the GPU's own parameters before it and its own raw gradients after it (the SGD kernel scales
them on the fly and never writes them back), so forward / backward rounding never accumulates: only the rule is under
test.  The model keeps its own float64 velocity.  Below that, the three kernels of the rule (w2l_sgd_step_ex,
w2l_finite_guard, w2l_sq_norm_accumulate) are checked one by one."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F, B, L = 16, 4, 10
ARCH = """V -1 NFEAT 1 0
C2 1 8 5 1 2 1 -1 -1
R
DO 0.0
LN 3
V 0 128 1 0
RO 1 0 3 2
L 128 NLABEL
"""
# short and long utterances in turn: with scale mode "none" the long batches' gradient norm is about 3x the short ones',
# so a clip threshold between the two binds on some steps only
T_STEPS = [120, 360, 120, 360, 120, 360]
ULP = 2.0 ** -24
# The kernel forms the update with at most 9 float32 roundings per step (1 / total_batch, the norm's cast and sqrt, its
# scaling, + 1e-6, the clip ratio, the scale product, g * scale, the momentum fma), each within ULP of a term bounded by
# V = mu V' + |G s c|, the float64 sum of magnitudes that forms v.  EPS = 16 ULP per step covers them; the velocity's
# error decays by mu < 1 each step and V_k >= mu^(k-j) V_j, so after step k it is within (k + 1) EPS V_k.
EPS = 16 * ULP


def f32(x):
    return float(np.float32(x))


def make_batch(N, criterion, T, seed, bad_token=False):
    rng = np.random.default_rng(seed)
    feat = torch.from_numpy(rng.normal(0, 1, (B, 1, F, T)).astype(np.float32)).cuda()
    y = rng.integers(0, N - 1 if criterion == "ctc" else N, (B, L)).astype(np.int32)  # ctc: blank = N - 1
    y[1, 6:] = -1
    if bad_token:
        y[2, 3] = N  # not a token: the criterion gives this sample a NaN loss
    return feat, torch.from_numpy(y).cuda()


def grads(tr):
    return tr.get_flat(0, 1).double(), tr.get_flat(1, 1).double()


def values(tr):
    return tr.get_flat(0, 0).clone(), tr.get_flat(1, 0).clone()


def scaled_norm(G, Gc, clamp_crit, s):
    sq = float((G * G).sum()) + (float((Gc * Gc).sum()) if clamp_crit else 0.0)
    return math.sqrt(sq) * s


def clip_factor(ns, M):
    return M / (ns + 1e-6) if M > 0 and ns > M else 1.0


class Rule:
    """float64 model of one update; keeps the velocity v and its magnitude sum V"""

    def __init__(self, lr, lrcrit, mu, M, total_batch, clamp_crit):
        self.lr, self.lrcrit, self.mu, self.M = f32(lr), f32(lrcrit), f32(mu), f32(M)  # what the kernels are given
        self.s = 1.0 / f32(total_batch)
        self.clamp_crit = clamp_crit
        self.v = self.V = None

    def step(self, p, t, G, Gc):
        ns = scaled_norm(G, Gc, self.clamp_crit, self.s)
        c = clip_factor(ns, self.M)
        g = G * (self.s * c)
        if self.v is None:
            self.v, self.V = torch.zeros_like(p), torch.zeros_like(p)
        self.v = self.mu * self.v + g
        self.V = self.mu * self.V + g.abs()
        u = Gc * (self.s * (c if self.clamp_crit else 1.0))
        return p - self.lr * self.v, t - self.lrcrit * u, u, ns, c


def check_close(name, got, want, before, tol, update):
    err = (got - want).abs()
    if bool((err <= tol).all()):
        return
    upd = before - got
    sel = update.abs() > 100 * tol
    factor = float((upd[sel] / update[sel]).median()) if bool(sel.any()) else float("nan")
    i = int((err - tol).argmax())
    raise AssertionError(f"{name}: element {i} off by {float(err[i]):.3e} > {float(tol[i]):.3e}; "
                         f"the applied update is {factor:.6f} x the model's (median over the elements)")


def probe(criterion, N, total_batch, batches):
    """gradient norms of the batches at the initial parameters (lr = 0, no clip), and the initial parameters"""
    from wav2letter_b200.trainer import Trainer

    tr = Trainer(ARCH, F, N, criterion, "none", transdiag=2.0, precision="f32", lr=0.0, lrcrit=0.0)
    p0, t0 = values(tr)
    s, clamp = 1.0 / f32(total_batch), criterion != "linseg"
    ns, G0 = [], None
    for feat, tgt in batches:
        tr.step(feat, tgt, total_batch=total_batch)
        G, Gc = grads(tr)
        G0 = (G, Gc) if G0 is None else G0
        ns.append(scaled_norm(G, Gc, clamp, s))
    assert torch.equal(tr.get_flat(0, 0), p0)
    tr.close()
    return p0, t0, ns, G0


def pick_rates(p0, t0, G0, s, c0, clamp_crit):
    """learning rates that move the network's median element and the transitions' norm by about 1 % on the first step:
    visible, and stable for six steps"""
    G, Gc = G0
    g = (G * s * c0).abs()
    lr = 0.01 * float(p0.double().abs().median()) / float(g[g > 0].median())
    if Gc.numel() == 0:
        return lr, 0.0
    return lr, 0.01 * float(t0.double().norm()) / float((Gc * s * (c0 if clamp_crit else 1.0)).norm())


def train_and_check(tr, rule, batches, total_batch, criterion):
    """one step per batch, each checked against the rule from the GPU's own values; returns the clipped steps"""
    clipped = []
    for k, (feat, tgt) in enumerate(batches):
        p, t = (x.double() for x in values(tr))
        tr.step(feat, tgt, total_batch=total_batch)
        G, Gc = grads(tr)
        p1, t1 = (x.double() for x in values(tr))
        pm, tm, u, ns, c = rule.step(p, t, G, Gc)
        if rule.M > 0:
            assert abs(ns / rule.M - 1) > 1e-3, f"step {k}: the norm {ns} is too close to the threshold to tell"
        clipped.append(c < 1.0)
        # the velocity's error, plus the roundings of lr * v and of the subtraction
        tol = 2 * ULP * torch.maximum(p.abs(), pm.abs()) + rule.lr * (k + 2) * EPS * rule.V
        check_close(f"step {k} network", p1, pm, p, tol, p - pm)
        # the update is visible: without this the check passes for any rule
        assert float((rule.lr * rule.v).abs().median()) >= 1e-3 * float(p.abs().median()), f"step {k}: update too small"
        if Gc.numel():
            tolc = 2 * ULP * torch.maximum(t.abs(), tm.abs()) + rule.lrcrit * 2 * EPS * u.abs()
            check_close(f"step {k} transitions", t1, tm, t, tolc, t - tm)
            # in norm: the transitions' gradient spans orders of magnitude, most entries of the FCC term are tiny
            assert rule.lrcrit * float(u.norm()) >= 1e-3 * float(t.norm()), f"step {k}: the transitions barely move"
        if criterion == "linseg":  # the criterion is large enough that leaving it out of the norm makes a difference
            assert float(Gc.norm()) >= 0.1 * float(G.norm()), (k, float(Gc.norm()), float(G.norm()))
    return clipped


# (criterion, N, momentum, clip regime, total_batch in units of B): a covering set, not the product.  asg / linseg at
# N = 8 take the 32-wide criterion calls, at N = 39 the 64-wide ones (N^2 not a multiple of 4).
CASES = [
    ("ctc", 12, 0.9, "some", 1), ("ctc", 12, 0.0, "every", 3), ("ctc", 12, 0.9, "off", 3), ("ctc", 12, 0.0, "never", 1),
    ("asg", 8, 0.9, "every", 1), ("asg", 8, 0.0, "some", 3), ("asg", 8, 0.9, "never", 1),
    ("asg", 39, 0.9, "some", 3), ("asg", 39, 0.0, "off", 1),
    ("linseg", 8, 0.9, "every", 3), ("linseg", 8, 0.0, "some", 1), ("linseg", 8, 0.9, "never", 3),
    ("linseg", 39, 0.9, "some", 1), ("linseg", 39, 0.0, "every", 3), ("linseg", 39, 0.9, "off", 1),
]


@pytest.mark.parametrize("criterion,N,momentum,regime,tb_mult", CASES)
def test_trainer_steps_follow_the_rule(criterion, N, momentum, regime, tb_mult):
    from wav2letter_b200.trainer import Trainer

    total_batch = float(B * tb_mult)  # 3 B: one rank of three
    clamp = criterion != "linseg"
    batches = [make_batch(N, criterion, T, 100 * N + k) for k, T in enumerate(T_STEPS)]
    p0, t0, ns, G0 = probe(criterion, N, total_batch, batches)
    short, long_ = ns[0::2], ns[1::2]
    assert 1.5 * max(short) < min(long_), ns
    # the norms drift as the model trains (by up to 2.5x over the six steps with momentum): "every" and "never" keep a
    # factor 10 from them, "some" sits between the short and the long batches
    M = {"off": 0.0, "never": 10 * max(ns), "every": 0.1 * min(ns), "some": math.sqrt(max(short) * min(long_))}[regime]
    s = 1.0 / f32(total_batch)
    lr, lrcrit = pick_rates(p0, t0, G0, s, clip_factor(ns[0], f32(M)), clamp)
    tr = Trainer(ARCH, F, N, criterion, "none", transdiag=2.0, lr=lr, lrcrit=lrcrit, momentum=momentum, maxgradnorm=M,
                 precision="f32")
    tr.set_flat(p0, 0)
    if t0.numel():
        tr.set_flat(t0, 1)
    clipped = train_and_check(tr, Rule(lr, lrcrit, momentum, M, total_batch, clamp), batches, total_batch, criterion)
    want = {"off": "none", "never": "none", "every": "all", "some": "some"}[regime]
    got = "none" if not any(clipped) else "all" if all(clipped) else "some"
    assert got == want, (regime, clipped)
    assert tr.skipped_steps() == 0
    tr.close()


@pytest.mark.parametrize("criterion", ["asg", "linseg"])
def test_guard_skips_a_step_with_a_nan_loss(criterion):
    """a sample whose target holds a token the criterion does not have gets a NaN loss: the whole update is skipped,
    velocity included, and counted; an eval step with a NaN loss is not counted"""
    from wav2letter_b200.trainer import Trainer

    N, mu = 8, 0.9
    clamp = criterion != "linseg"
    good = [make_batch(N, criterion, T, 700 + k) for k, T in enumerate([120, 360, 360])]
    bad = make_batch(N, criterion, 120, 710, bad_token=True)
    p0, t0, ns, G0 = probe(criterion, N, B, good)
    M = 0.5 * min(ns)
    lr, lrcrit = pick_rates(p0, t0, G0, 1.0 / B, clip_factor(ns[0], f32(M)), clamp)
    tr = Trainer(ARCH, F, N, criterion, "none", transdiag=2.0, lr=lr, lrcrit=lrcrit, momentum=mu, maxgradnorm=M, precision="f32")
    tr.set_flat(p0, 0)
    tr.set_flat(t0, 1)
    rule = Rule(lr, lrcrit, mu, M, B, clamp)
    train_and_check(tr, rule, good[:2], B, criterion)
    assert tr.skipped_steps() == 0
    before = values(tr)
    loss = tr.step(*bad, total_batch=B)
    after = values(tr)
    assert torch.isnan(loss[2]) and torch.isfinite(loss[[0, 1, 3]]).all()
    assert torch.equal(after[0], before[0]) and torch.equal(after[1], before[1])
    assert tr.skipped_steps() == 1
    # the next good step continues from the velocity of before the bad step (the model never saw the bad one)
    p, t = (x.double() for x in before)
    tr.step(*good[2], total_batch=B)
    G, Gc = grads(tr)
    pm, tm, u, _, _ = rule.step(p, t, G, Gc)
    p1, t1 = (x.double() for x in values(tr))
    check_close("after the skipped step, network", p1, pm, p, 2 * ULP * torch.maximum(p.abs(), pm.abs()) + rule.lr * 4 * EPS * rule.V, p - pm)
    check_close("after the skipped step, transitions", t1, tm, t, 2 * ULP * torch.maximum(t.abs(), tm.abs()) + rule.lrcrit * 2 * EPS * u.abs(), t - tm)
    assert tr.skipped_steps() == 1
    loss = tr.step(*bad, train=False)
    assert torch.isnan(loss[2]) and tr.skipped_steps() == 1
    tr.close()


@pytest.mark.parametrize("total_batch", [0.0, -1.0, float("nan"), float("inf")])
def test_training_step_rejects_a_bad_total_batch(total_batch):
    from wav2letter_b200 import W2LError
    from wav2letter_b200.trainer import Trainer

    N = 8
    tr = Trainer(ARCH, F, N, "asg", "none", transdiag=2.0, lr=0.01, lrcrit=0.01, momentum=0.9, maxgradnorm=1.0, precision="f32")
    feat, tgt = make_batch(N, "asg", 120, 900)
    tr.step(feat, tgt)  # a velocity, so that even a zero gradient scale (total_batch = inf) would move the parameters
    before = values(tr)
    with pytest.raises(W2LError) as e:
        tr.step(feat, tgt, train=True, total_batch=total_batch)
    assert e.value.code == 1
    after = values(tr)
    assert torch.equal(after[0], before[0]) and torch.equal(after[1], before[1])
    assert tr.skipped_steps() == 0
    loss = tr.step(feat, tgt, train=False, total_batch=total_batch)  # an eval step does not use total_batch
    assert torch.isfinite(loss).all()
    assert torch.equal(values(tr)[0], before[0])
    tr.close()


# ---- the kernels ------------------------------------------------------------------------------------------------------

def _lib():
    from wav2letter_b200 import capi

    return capi


def sgd_ref(p, g, v, lr, mu, wd, gs, M, sq, nesterov):
    """float64 w2l_sgd_step_ex; returns (p', v', the magnitude sum behind v', the one behind the step)"""
    scale = gs
    if M > 0 and sq is not None:
        nrm = math.sqrt(sq) * gs
        if nrm > M:
            scale *= M / (nrm + 1e-6)
    gi = g * scale + wd * p
    mag = (g * scale).abs() + wd * p.abs()
    if mu == 0:
        return p - lr * gi, v, mag, mag
    v1 = mu * v + gi
    V = mu * v.abs() + mag
    if nesterov:
        return p - lr * (gi + mu * v1), v1, V, mag + mu * V
    return p - lr * v1, v1, V, V


@pytest.mark.parametrize("n", [1, 3, 257, (1 << 20) + 5])
@pytest.mark.parametrize("mode", ["sgd", "momentum", "nesterov"])
def test_sgd_step_ex_matches_float64(n, mode):
    capi = _lib()
    g = torch.Generator(device="cuda").manual_seed(n)
    p0 = torch.randn(n, device="cuda", generator=g)
    gr = torch.randn(n, device="cuda", generator=g) * 3
    v0 = torch.randn(n, device="cuda", generator=g)
    sq = float((gr.double() ** 2).sum())
    lr, mu, nesterov = f32(0.1), (0.0 if mode == "sgd" else f32(0.9)), int(mode == "nesterov")
    for wd in (0.0, f32(1e-2)):
        for gs in (1.0, f32(1 / 48)):
            nrm = math.sqrt(sq) * gs
            for clip in ("off", "binding", "loose", "null_sq"):
                M = {"off": 0.0, "binding": f32(0.5 * nrm), "loose": f32(2 * nrm), "null_sq": f32(0.5 * nrm)}[clip]
                sq_dev = None if clip == "null_sq" else torch.tensor([sq], dtype=torch.float64, device="cuda")
                for guard in (None, 0, 1):
                    gd = None if guard is None else torch.tensor([guard, 7], dtype=torch.int32, device="cuda")
                    p, v = p0.clone(), v0.clone()
                    capi._check(capi.lib.w2l_sgd_step_ex(capi._stream(), n, capi._ptr(p), capi._ptr(gr), capi._ptr(v), lr, mu, wd, gs,
                                                         M, capi._ptr(sq_dev), nesterov, capi._ptr(gd)))
                    torch.cuda.synchronize()
                    where = f"wd={wd} gs={gs} clip={clip} guard={guard}"
                    if guard == 1:
                        assert torch.equal(p, p0) and torch.equal(v, v0), where
                        continue
                    pr, vr, Vv, Vp = sgd_ref(p0.double(), gr.double(), v0.double(), lr, mu, wd, gs, M, None if clip == "null_sq" else sq,
                                             nesterov)
                    if mu == 0:
                        assert torch.equal(v, v0), where
                    else:
                        assert bool(((v.double() - vr).abs() <= EPS * Vv).all()), where
                    assert bool(((p.double() - pr).abs() <= 2 * ULP * pr.abs() + lr * 2 * EPS * Vp).all()), where
                    assert gd is None or gd.tolist() == [0, 7], where


FINITE_GUARD_CASES = [  # (bad loss index or None, its value, *sq_norm or None for a null pointer, n_loss, expected bad)
    (None, 0.0, 3.0, 1000, False),
    (0, float("nan"), 3.0, 1000, True), (999, float("nan"), 3.0, 1000, True),
    (0, float("inf"), 3.0, 1000, True), (999, -float("inf"), 3.0, 1000, True),
    (None, 0.0, float("nan"), 1000, True), (None, 0.0, float("inf"), 1000, True),
    (None, 0.0, None, 1000, False), (999, float("nan"), None, 1000, True),
    (None, 0.0, 3.0, 0, False), (None, 0.0, float("nan"), 0, True),
]


@pytest.mark.parametrize("bad_at,value,sq,n_loss,bad", FINITE_GUARD_CASES)
def test_finite_guard(bad_at, value, sq, n_loss, bad):
    capi = _lib()
    loss = torch.rand(1000, device="cuda") * 50
    if bad_at is not None:
        loss[bad_at] = value
    sq_dev = None if sq is None else torch.tensor([sq], dtype=torch.float64, device="cuda")
    guard = torch.tensor([1, 5], dtype=torch.int32, device="cuda")  # guard[0] left set by an earlier bad step
    capi._check(capi.lib.w2l_finite_guard(capi._stream(), n_loss, capi._ptr(loss) if n_loss else None, capi._ptr(sq_dev), capi._ptr(guard)))
    assert guard.tolist() == ([1, 6] if bad else [0, 5])


def test_finite_guard_counts_across_calls():
    capi = _lib()
    guard = torch.zeros(2, dtype=torch.int32, device="cuda")
    good, nan = torch.ones(3, device="cuda"), torch.tensor([1.0, float("nan"), 1.0], device="cuda")
    seen = []
    for loss in (nan, good, nan, nan, good):
        capi._check(capi.lib.w2l_finite_guard(capi._stream(), 3, capi._ptr(loss), None, capi._ptr(guard)))
        seen.append(guard.tolist())
    assert seen == [[1, 1], [0, 1], [1, 2], [1, 3], [0, 3]]


@pytest.mark.parametrize("n", [1, 3, 257, 2049, (1 << 20) + 5])
def test_sq_norm_accumulate(n):
    capi = _lib()
    g = torch.randn(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(n)) * 7
    out = torch.tensor([5.0], dtype=torch.float64, device="cuda")
    capi._check(capi.lib.w2l_sq_norm_accumulate(capi._stream(), n, capi._ptr(g), capi._ptr(out)))
    want = 5.0 + float((g.double() ** 2).sum())
    assert abs(out.item() - want) <= 1e-12 * want
    runs = []
    for _ in range(2):
        o = torch.zeros(1, dtype=torch.float64, device="cuda")
        capi._check(capi.lib.w2l_sq_norm_accumulate(capi._stream(), n, capi._ptr(g), capi._ptr(o)))
        runs.append(o.clone())
    assert torch.equal(runs[0], runs[1])
