"""The streaming acoustic model in fp16 precision: the chunking and batching invariance of test_gpu_streaming.py (the
split of an utterance into chunks, and the number of streams in a call, do not change a bit of its emissions)."""
import pytest

import test_gpu_streaming as base

pytestmark = pytest.mark.gpu


def test_chunking_does_not_change_a_bit_fp16():
    base.test_chunking_does_not_change_a_bit("fp16")


def test_large_batches_equal_single_stream_runs_fp16():
    base.test_large_batches_equal_single_stream_runs("fp16")
