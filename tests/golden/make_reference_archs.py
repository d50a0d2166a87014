"""Stores the token streams of the reference's arch files (wav2letter_b200/archs.py REFERENCE_FILES) in
tests/golden/reference_archs.json, the data tests/test_archs.py compares the generators against.

    python tests/golden/make_reference_archs.py <root of the reference wav2letter tree>"""
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location("w2l_archs", os.path.join(HERE, "..", "..", "wav2letter_b200", "archs.py"))
archs = importlib.util.module_from_spec(spec)
spec.loader.exec_module(archs)


def tokens(text):
    return [ln.split("#")[0].split() for ln in text.splitlines() if ln.split("#")[0].split()]


def main(ref_root):
    out = {name: {"file": rel, "tokens": tokens(open(os.path.join(ref_root, rel)).read())}
           for name, rel in sorted(archs.REFERENCE_FILES.items())}
    with open(os.path.join(HERE, "reference_archs.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
