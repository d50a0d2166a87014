"""Trainer.step(..., text=...) checks its arguments before anything runs: a TextPipeline, a training step, no seq2seq
sizes, a text pipeline of the trainer's criterion and a [B, L] target.  The trainer here has no handle and the tensors
live on the host, so a check that let a call through would fail differently.  Nothing here reaches a GPU."""
import pytest
import torch


def _trainer(criterion):
    from wav2letter_b200.trainer import Trainer

    tr = Trainer.__new__(Trainer)
    tr.h, tr.criterion = None, criterion
    return tr


def _text(criterion):
    from wav2letter_b200.text import TextPipeline

    return TextPipeline("|\na\nb\n", "", criterion, 0, "", False, "|")


FEAT = torch.zeros((2, 1, 4, 8))
TGT = torch.zeros((2, 3), dtype=torch.int32)


@pytest.mark.parametrize("kwargs,error", [
    (dict(text="ctc"), TypeError),
    (dict(train=False), ValueError),
    (dict(input_sizes=[8, 8]), ValueError),
    (dict(target_sizes=[3, 3]), ValueError),
])
def test_scored_step_arguments(kwargs, error):
    kw = dict(text=_text("ctc"))
    kw.update(kwargs)
    with pytest.raises(error):
        _trainer("ctc").step(FEAT, TGT, **kw)


@pytest.mark.parametrize("trainer,text", [("ctc", "asg"), ("asg", "ctc"), ("linseg", "ctc"), ("seq2seq", "seq2seq")])
def test_text_pipeline_of_another_criterion_is_refused(trainer, text):
    with pytest.raises(ValueError):
        _trainer(trainer).step(FEAT, TGT, text=_text(text))


@pytest.mark.parametrize("target", [torch.zeros((3, 3), dtype=torch.int32), torch.zeros(6, dtype=torch.int32)])
def test_target_rows_must_match_the_batch(target):
    with pytest.raises(ValueError):
        _trainer("linseg").step(FEAT, target, text=_text("asg"))


def test_matching_arguments_reach_the_device_checks():
    # every check above passes; the host tensors are then refused as not CUDA
    with pytest.raises(TypeError, match="CUDA"):
        _trainer("asg").step(FEAT, TGT, text=_text("asg"))
