#!/usr/bin/env python3
"""Write tests/golden/bls_sign_kat.json: the Ethereum BLS signing and aggregation vectors the suite checks.

  python tests/golden/make_bls_sign_golden.py <constantine checkout>

Sources (inside the checkout), copied verbatim with nothing computed:
  tests/protocol_blssig_pop_on_bls12381_g2_test_vectors_v0.1.1/sign/*.json        10 vectors: privkey, message -> signature or null
  tests/protocol_blssig_pop_on_bls12381_g2_test_vectors_v0.1.1/aggregate/*.json    6 vectors: signatures -> their sum or null
"""
import glob
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
COUNTS = {"sign": 10, "aggregate": 6}


def main(checkout):
    base = os.path.join(checkout, "tests", "protocol_blssig_pop_on_bls12381_g2_test_vectors_v0.1.1")
    out = {}
    for kind, count in COUNTS.items():
        vectors = []
        for path in sorted(glob.glob(os.path.join(base, kind, "*.json"))):
            with open(path) as f:
                v = json.load(f)
            vectors.append({"name": os.path.splitext(os.path.basename(path))[0], "input": v["input"], "output": v["output"]})
        assert len(vectors) == count, (kind, len(vectors))
        out[kind] = vectors
    with open(os.path.join(HERE, "bls_sign_kat.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
