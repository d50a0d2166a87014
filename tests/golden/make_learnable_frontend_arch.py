"""Stores the token stream of the TIMIT recipe's arch file (wav2letter_b200/archs.py LEARNABLE_FRONTEND_FILE) in
tests/golden/learnable_frontend_arch.json, the data tests/test_archs_learnable_frontend.py compares the generator against.

    python tests/golden/make_learnable_frontend_arch.py <root of the reference wav2letter tree>"""
import json
import os
import sys

from make_reference_archs import archs, tokens

HERE = os.path.dirname(os.path.abspath(__file__))


def main(ref_root):
    rel = archs.LEARNABLE_FRONTEND_FILE
    with open(os.path.join(HERE, "learnable_frontend_arch.json"), "w") as f:
        json.dump({"file": rel, "tokens": tokens(open(os.path.join(ref_root, rel)).read())}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
