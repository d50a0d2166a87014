"""The arch generators of wav2letter_b200/archs.py reproduce the reference's arch files token for token (the reference
files' token streams are stored in tests/golden/reference_archs.json by tests/golden/make_reference_archs.py)."""
import importlib.util
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("w2l_archs", os.path.join(ROOT, "wav2letter_b200", "archs.py"))
archs = importlib.util.module_from_spec(spec)
spec.loader.exec_module(archs)

with open(os.path.join(ROOT, "tests", "golden", "reference_archs.json")) as _f:
    GOLDEN = json.load(_f)


def tokens(text):
    return [ln.split("#")[0].split() for ln in text.splitlines() if ln.split("#")[0].split()]


@pytest.mark.parametrize("name", sorted(archs.REFERENCE_FILES))
def test_generated_arch_matches_reference_file(name):
    assert GOLDEN[name]["file"] == archs.REFERENCE_FILES[name]
    gen = archs.BASELINE_ARCHS[name][0]
    text = gen(ctc_head=False) if name == "seq2seq_tds_ctc" else gen()
    assert tokens(text) == GOLDEN[name]["tokens"]


def test_ctc_head_only_changes_the_last_linear():
    a, b = tokens(archs.seq2seq_tds(True)), tokens(archs.seq2seq_tds(False))
    assert a[:-1] == b[:-1] and a[-1] == ["L", "1440", "NLABEL"] and b[-1] == ["L", "1440", "1024"]
