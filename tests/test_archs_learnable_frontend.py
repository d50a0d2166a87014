"""learnable_frontend_timit() reproduces the TIMIT recipe's arch file token for token (its token stream is stored in
tests/golden/learnable_frontend_arch.json by tests/golden/make_learnable_frontend_arch.py), and stays out of the
BASELINE tables that bench.py and test_archs.py walk."""
import importlib.util
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("w2l_archs", os.path.join(ROOT, "wav2letter_b200", "archs.py"))
archs = importlib.util.module_from_spec(spec)
spec.loader.exec_module(archs)


def tokens(text):
    return [ln.split("#")[0].split() for ln in text.splitlines() if ln.split("#")[0].split()]


def test_generated_arch_matches_reference_file():
    with open(os.path.join(ROOT, "tests", "golden", "learnable_frontend_arch.json")) as f:
        golden = json.load(f)
    assert golden["file"] == archs.LEARNABLE_FRONTEND_FILE
    assert tokens(archs.learnable_frontend_timit()) == golden["tokens"]


def test_not_a_baseline_arch():
    assert all(gen is not archs.learnable_frontend_timit for gen, *_ in archs.BASELINE_ARCHS.values())
    assert archs.LEARNABLE_FRONTEND_FILE not in archs.REFERENCE_FILES.values()
