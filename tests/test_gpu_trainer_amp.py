"""Dynamic loss scaling in the trainer (w2l_trainer_set_amp) against a float64 model of Train.cpp's rule
(:1135-1140, 1681-1684, 1748-1790, 1806-1818):

    every attempt:   counter = (counter + 1) mod 2^16                  (unsigned short)
    loss finite, gradient not, scale >= min_scale:  scale /= 2, counter = 1, run the same batch again
    gradient not finite otherwise:                  counter = 1, the update is skipped
    after the step, if scale < max_scale:           scale = 2 scale if counter % interval == 0 else scale + 2

The loss gradient carries the scale and the update divides it out.  An initial scale large enough that the fp16 GEMM
operands of the backward overflow (a numeric Inf, caught by the finite guard) makes the trainer retry; the scales,
counters and retries must follow the model, and the parameters after the retried step must equal, bit for bit, those of a
fresh trainer started at the final scale.  A checkpoint keeps the loss-scaling state, and a run resumed from it continues
bit for bit."""
import pytest
import torch

import test_gpu_optimizer_step as opt

pytestmark = pytest.mark.gpu

N, CRIT = 8, "asg"


class AmpModel:
    def __init__(self, scale, interval, max_scale, min_scale):
        self.scale, self.interval, self.max_scale, self.min_scale = float(scale), interval, float(max_scale), float(min_scale)
        self.counter, self.retries = 1, 0

    def step(self, overflows):
        """one training step whose first `overflows` attempts have a non-finite gradient; returns whether it updated"""
        bad = overflows
        while True:
            self.counter = (self.counter + 1) % 65536
            if bad > 0:
                bad -= 1
                if self.scale >= self.min_scale:
                    self.scale /= 2.0
                    self.counter = 1
                    self.retries += 1
                    continue
                self.counter = 1
                updated = False
            else:
                updated = True
            break
        if self.scale < self.max_scale:
            self.scale = self.scale * 2 if self.counter % self.interval == 0 else self.scale + 2
        return updated

    def state(self):
        return self.scale, self.counter, self.retries


def _trainer(precision, lr=0.005, lrcrit=0.001, momentum=0.5):
    from wav2letter_b200.trainer import Trainer

    return Trainer(opt.ARCH, opt.F, N, CRIT, "none", transdiag=2.0, lr=lr, lrcrit=lrcrit, momentum=momentum, precision=precision)


def _batches(seed, n=6):
    return [opt.make_batch(N, CRIT, T, seed + k) for k, T in enumerate(opt.T_STEPS[:n])]


def test_scale_grows_by_the_rule_and_the_update_divides_it_out():
    """no overflow: +2 per step, x2 every `interval` attempts, capped at max_scale; the raw gradients carry the scale
    and every update follows the SGD rule with the gradients divided by total_batch * scale"""
    batches = _batches(40)
    # rates that move the parameters by about 1 % per step (test_gpu_optimizer_step.py): visible and stable
    p0, t0, _, G0 = opt.probe(CRIT, N, float(opt.B), batches)
    lr, lrcrit = opt.pick_rates(p0, t0, G0, 1.0 / opt.f32(opt.B), 1.0, True)
    plain = _trainer("f32", lr, lrcrit, 0.9)
    tr = _trainer("f32", lr, lrcrit, 0.9)
    for t in (plain, tr):
        t.set_flat(p0, 0)
        t.set_flat(t0, 1)
    tr.set_amp(True, initial_scale=8.0, update_interval=2, max_scale=20.0, min_scale=1e-4)
    model = AmpModel(8.0, 2, 20.0, 1e-4)
    rule = opt.Rule(lr, lrcrit, 0.9, 0.0, float(opt.B), True)
    for k, (feat, tgt) in enumerate(batches):
        scale = model.scale
        p, t = (x.double() for x in opt.values(tr))
        tr.step(feat, tgt)
        model.step(0)
        assert tr.amp_state() == model.state(), (k, tr.amp_state(), model.state())
        G, Gc = opt.grads(tr)
        if k == 0:  # the same parameters without loss scaling: the gradients differ by the scale
            plain.step(feat, tgt)
            Gp, Gcp = opt.grads(plain)
            assert float((G / opt.f32(scale) - Gp).abs().max()) <= 1e-5 * float(Gp.abs().max())
            assert float((Gc / opt.f32(scale) - Gcp).abs().max()) <= 1e-5 * float(Gcp.abs().max())
        rule.s = 1.0 / (float(opt.B) * scale)
        pm, tm, u, _, _ = rule.step(p, t, G, Gc)
        p1, t1 = (x.double() for x in opt.values(tr))
        tol = 2 * opt.ULP * torch.maximum(p.abs(), pm.abs()) + rule.lr * (k + 2) * opt.EPS * rule.V
        opt.check_close(f"step {k} network", p1, pm, p, tol, p - pm)
        tolc = 2 * opt.ULP * torch.maximum(t.abs(), tm.abs()) + rule.lrcrit * 2 * opt.EPS * u.abs()
        opt.check_close(f"step {k} transitions", t1, tm, t, tolc, t - tm)
    assert model.scale >= 20.0  # the cap was reached
    assert tr.skipped_steps() == 0
    tr.close()
    plain.close()


def test_overflowing_scale_retries_and_equals_a_fresh_trainer_at_the_final_scale():
    s0 = 2.0 ** 40
    batches = _batches(70, 4)
    tr = _trainer("fp16")
    p0, t0 = opt.values(tr)
    tr.set_amp(True, initial_scale=s0)
    model = AmpModel(s0, 2000, 32000.0, 1e-4)
    final_scales = []
    for k, (feat, tgt) in enumerate(batches):
        before = tr.amp_state()
        tr.step(feat, tgt)
        if k == 0:
            after_first = opt.values(tr)
        retried = tr.amp_state()[2] - before[2]
        final_scales.append(before[0] / 2.0 ** retried)
        model.step(retried)
        assert tr.amp_state() == model.state(), (k, tr.amp_state(), model.state())
    assert final_scales[0] < s0 / 2 ** 10  # fp16 gradients of 2^40 times the loss overflow: many retries
    assert tr.skipped_steps() == 0
    tr.close()
    # a fresh trainer at the last scale that overflowed overflows too; one at the final scale does not, and its update
    # equals the retried step's bit for bit
    feat, tgt = batches[0]
    for scale, retries in ((2 * final_scales[0], 1), (final_scales[0], 0)):
        fresh = _trainer("fp16")
        fresh.set_flat(p0, 0)
        fresh.set_flat(t0, 1)
        fresh.set_amp(True, initial_scale=scale)
        fresh.step(feat, tgt)
        assert (fresh.amp_state()[2] > 0) == (retries > 0), (scale, fresh.amp_state())
        if retries == 0:
            got = opt.values(fresh)
            assert torch.equal(got[0], after_first[0]) and torch.equal(got[1], after_first[1])
        fresh.close()


def test_below_min_scale_the_step_is_skipped_not_retried():
    feat, tgt = _batches(90, 1)[0]
    tr = _trainer("fp16")
    before = opt.values(tr)
    tr.set_amp(True, initial_scale=2.0 ** 40, min_scale=2.0 ** 41)
    tr.step(feat, tgt)
    model = AmpModel(2.0 ** 40, 2000, 32000.0, 2.0 ** 41)
    assert model.step(1) is False
    assert tr.amp_state() == model.state() == (2.0 ** 40, 1, 0)
    assert tr.skipped_steps() == 1
    after = opt.values(tr)
    assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1])
    tr.close()


def test_checkpoint_keeps_the_loss_scaling_state(tmp_path):
    from wav2letter_b200.trainer import Trainer

    batches = _batches(110)
    tr = _trainer("fp16")
    tr.set_amp(True, initial_scale=2.0 ** 30, update_interval=3, max_scale=2.0 ** 31)
    for feat, tgt in batches[:3]:
        tr.step(feat, tgt)
    state = tr.amp_state()
    assert state[2] > 0  # the run has retried
    path = str(tmp_path / "amp.ckpt")
    tr.save(path)
    for feat, tgt in batches[3:]:
        tr.step(feat, tgt)
    want, want_state = opt.values(tr), tr.amp_state()
    tr.close()
    tr2 = Trainer.load(path)
    assert tr2.amp_state() == state
    for feat, tgt in batches[3:]:
        tr2.step(feat, tgt)
    got = opt.values(tr2)
    assert tr2.amp_state() == want_state
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    tr2.close()


def test_loss_scaling_off_changes_nothing():
    """set_amp(False) after a run with it: the same bits as a trainer that never had it"""
    batches = _batches(130, 2)
    a, b = _trainer("bf16"), _trainer("bf16")
    b.set_flat(opt.values(a)[0], 0)
    b.set_flat(opt.values(a)[1], 1)
    b.set_amp(True, initial_scale=64.0)
    b.set_amp(False)
    for feat, tgt in batches:
        a.step(feat, tgt)
        b.step(feat, tgt)
    va, vb = opt.values(a), opt.values(b)
    assert torch.equal(va[0], vb[0]) and torch.equal(va[1], vb[1])
    a.close()
    b.close()
