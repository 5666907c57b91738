"""Regenerate tests/golden/seam_v1.json: the types of the members, constants and globals of the reference's interface that
tools/integration_stub.cpp reads (and the constants' values), as the reference's own headers declare them.

  python tests/golden/make_seam_golden.py <Cerberus checkout>/src
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from helpers import seam_probe          # noqa: E402

if __name__ == "__main__":
    if len(sys.argv) != 2 or not os.path.isdir(sys.argv[1]):
        sys.exit(__doc__)
    with tempfile.TemporaryDirectory() as tmp:
        facts = seam_probe(sys.argv[1], tmp)
    with open(os.path.join(HERE, "seam_v1.json"), "w") as f:
        json.dump(facts, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {os.path.join(HERE, 'seam_v1.json')}: {len(facts) - 1} declarations")
