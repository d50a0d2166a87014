"""The learning-rate schedule of Train.cpp:1169-1175, 1334-1348 in the trainer, against a float64 model:

    lr = initlr * 0.5^(curEpoch < lr_decay ? 0 : 1 + (curEpoch - lr_decay) // lr_decay_step)
                * (cos(pi/2 * curBatch / nbatches) if lrcosine else gamma^(curBatch / stepsize))
                * min(curBatch / warmup, 1)

with curBatch the 1-based number of the update (every training step counts, a skipped one too).  The rates the trainer
reports equal the model rounded to float32; every update of a run through warmup, gamma / stepsize, cosine and epoch
decay follows the SGD rule of test_gpu_optimizer_step.py at the model's rate for that update; a checkpoint taken mid-run
and loaded continues the run bit for bit; a checkpoint without the schedule (version 1) still loads."""
import math
import struct

import numpy as np
import pytest
import torch

import test_gpu_optimizer_step as opt

pytestmark = pytest.mark.gpu

INT64_MAX = (1 << 63) - 1
DEFAULT = dict(warmup=1, gamma=1.0, stepsize=INT64_MAX, lrcosine=False, nbatches=INT64_MAX, lr_decay=INT64_MAX,
               lr_decay_step=INT64_MAX)


def model_lr(lr0, cur_batch, epoch, warmup, gamma, stepsize, lrcosine, nbatches, lr_decay, lr_decay_step):
    after = epoch - lr_decay
    decay = math.pow(0.5, 0 if after < 0 else 1 + after // lr_decay_step)
    sched = math.cos(cur_batch / nbatches * math.acos(-1) / 2.0) if lrcosine else math.pow(gamma, cur_batch / stepsize)
    warm = min(cur_batch / warmup, 1.0) if warmup else 1.0  # Train.cpp: curBatch / 0.0 = inf
    return opt.f32(float(np.float32(lr0)) * decay * sched * warm)


SCHEDULES = [
    dict(DEFAULT),
    dict(DEFAULT, warmup=5),
    dict(DEFAULT, warmup=0, gamma=0.5, stepsize=40),  # seq2seq_tds/librispeech/train.cfg
    dict(DEFAULT, warmup=3, lrcosine=True, nbatches=20),
    dict(DEFAULT, lr_decay=2, lr_decay_step=3),
    dict(DEFAULT, warmup=4, gamma=0.8, stepsize=3, lr_decay=1, lr_decay_step=1),
]


def _trainer(lr=0.3, lrcrit=0.02, precision="f32", criterion="asg", N=8, momentum=0.9):
    from wav2letter_b200.trainer import Trainer

    return Trainer(opt.ARCH, opt.F, N, criterion, "none", transdiag=2.0, lr=lr, lrcrit=lrcrit, momentum=momentum,
                   precision=precision)


@pytest.mark.parametrize("sched", SCHEDULES)
def test_reported_rates_follow_the_formula(sched):
    tr = _trainer()
    tr.set_schedule(**sched)
    for update in (0, 1, 2, 4, 7, 19, 39, 40, 41, 100):
        for epoch in (0, 1, 2, 3, 5, 9):
            tr.set_position(update, epoch)
            assert tr.position() == (update, epoch)
            want = (model_lr(0.3, update + 1, epoch, **sched), model_lr(0.02, update + 1, epoch, **sched))
            assert tr.lr() == want, (sched, update, epoch, tr.lr(), want)
    tr.close()


def test_default_schedule_leaves_the_rates_alone_and_set_lr_replaces_them():
    tr = _trainer()
    tr.set_position(12345, 17)
    assert tr.lr() == (opt.f32(0.3), opt.f32(0.02))
    tr.set_lr(0.125, 0.5)
    assert tr.lr() == (0.125, 0.5)
    tr.set_schedule(warmup=4)
    tr.set_position(0, 1)
    assert tr.lr() == (0.125 / 4, 0.5 / 4)
    tr.close()


@pytest.mark.parametrize("sched", [dict(DEFAULT, warmup=3, gamma=0.5, stepsize=2, lr_decay=2, lr_decay_step=1),
                                   dict(DEFAULT, warmup=2, lrcosine=True, nbatches=8)])
def test_every_update_follows_the_rule_at_the_scheduled_rate(sched):
    """six updates over two epochs (the epoch changes after the third): each one from the GPU's own parameters and raw
    gradients, at the model's rate for that update; a step whose loss is NaN is skipped and still counts"""
    N, total_batch, criterion = 8, float(opt.B), "asg"
    batches = [opt.make_batch(N, criterion, T, 700 + k) for k, T in enumerate(opt.T_STEPS)]
    p0, t0, ns, G0 = opt.probe(criterion, N, total_batch, batches)
    lr0, lrcrit0 = opt.pick_rates(p0, t0, G0, 1.0 / opt.f32(total_batch), 1.0, True)
    lr0, lrcrit0 = 4 * lr0, 4 * lrcrit0  # the schedule scales them down
    tr = _trainer(lr=lr0, lrcrit=lrcrit0, criterion=criterion, N=N)
    tr.set_flat(p0, 0)
    tr.set_flat(t0, 1)
    tr.set_schedule(**sched)
    tr.set_position(0, 1)
    rule = opt.Rule(lr0, lrcrit0, 0.9, 0.0, total_batch, True)
    bad = opt.make_batch(N, criterion, 120, 1, bad_token=True)
    for k, (feat, tgt) in enumerate(batches):
        if k == 3:
            tr.set_position(tr.position()[0], 2)
        if k == 4:  # a skipped update: nothing moves, curBatch advances
            before = opt.values(tr)
            tr.step(*bad, total_batch=total_batch)
            assert all(torch.equal(a, b) for a, b in zip(before, opt.values(tr)))
        update, epoch = tr.position()
        rule.lr, rule.lrcrit = model_lr(lr0, update + 1, epoch, **sched), model_lr(lrcrit0, update + 1, epoch, **sched)
        assert tr.lr() == (rule.lr, rule.lrcrit)
        p, t = (x.double() for x in opt.values(tr))
        tr.step(feat, tgt, total_batch=total_batch)
        assert tr.position() == (update + 1, epoch)
        G, Gc = opt.grads(tr)
        p1, t1 = (x.double() for x in opt.values(tr))
        pm, tm, u, _, _ = rule.step(p, t, G, Gc)
        tol = 2 * opt.ULP * torch.maximum(p.abs(), pm.abs()) + rule.lr * (k + 2) * opt.EPS * rule.V
        opt.check_close(f"update {update + 1} network", p1, pm, p, tol, p - pm)
        tolc = 2 * opt.ULP * torch.maximum(t.abs(), tm.abs()) + rule.lrcrit * 2 * opt.EPS * u.abs()
        opt.check_close(f"update {update + 1} transitions", t1, tm, t, tolc, t - tm)
    assert tr.skipped_steps() == 1
    assert tr.position() == (len(batches) + 1, 2)
    tr.close()


def _run(tr, batches):
    for feat, tgt in batches:
        tr.step(feat, tgt)
    return opt.values(tr)


@pytest.mark.parametrize("precision", ["f32", "fp16"])
def test_checkpoint_mid_run_continues_bit_for_bit(tmp_path, precision):
    from wav2letter_b200.trainer import Trainer

    batches = [opt.make_batch(8, "asg", T, 900 + k) for k, T in enumerate(opt.T_STEPS)]
    tr = _trainer(lr=0.05, lrcrit=0.01, precision=precision)
    tr.set_schedule(warmup=2, gamma=0.7, stepsize=2, lr_decay=1, lr_decay_step=2)
    tr.set_position(10, 3)
    _run(tr, batches[:3])
    path = str(tmp_path / "mid.ckpt")
    tr.save(path)
    want = _run(tr, batches[3:])
    pos = tr.position()
    tr.close()
    tr2 = Trainer.load(path)
    assert tr2.position() == (13, 3)
    got = _run(tr2, batches[3:])
    assert tr2.position() == pos
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    tr2.close()


def test_version1_checkpoint_loads_without_schedule(tmp_path):
    """a version-1 file is a version-2 file without the trailing position, schedule and loss scaling"""
    from wav2letter_b200.trainer import Trainer

    tr = _trainer()
    tr.set_schedule(warmup=7, gamma=0.5, stepsize=3)
    tr.set_position(5, 2)
    tr.set_amp(True, initial_scale=256.0)
    path = tmp_path / "v2.ckpt"
    tr.save(str(path))
    want = opt.values(tr)
    tr.close()
    data = path.read_bytes()
    tail = 8 + 8 + 8 + 8 + 8 + 4 + 8 + 8 + 8  # update, epoch, warmup, gamma, stepsize, lrcosine, nbatches, lr_decay, lr_decay_step
    tail += 4 + 8 + 4 + 8 + 8 + 4 + 8  # loss scaling: on, scale, update_interval, max_scale, min_scale, counter, retries
    assert struct.unpack_from("<I", data, 8)[0] == 2
    v1 = data[:8] + struct.pack("<I", 1) + data[12:-tail]
    (tmp_path / "v1.ckpt").write_bytes(v1)
    tr1 = Trainer.load(str(tmp_path / "v1.ckpt"))
    assert tr1.position() == (0, 0)
    assert tr1.lr() == (opt.f32(0.3), opt.f32(0.02))
    assert tr1.amp_state() == (4096.0, 1, 0)
    got = opt.values(tr1)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    tr1.close()
