#!/usr/bin/env python3
"""Build tests/golden/evm_bn254_pairing_kat.json from the reference's EIP-197 ecPairing vectors (run where the reference tree
exists; the fixture -- not this script -- is what the tests read).

Source: reference tests/protocol_ethereum_evm_precompiles/bn256Pairing.json (14 vectors from the go-ethereum suite): per vector the
hex input (k x 192 bytes: P.x, P.y, Q.x_im, Q.x_re, Q.y_im, Q.y_re, 32-byte big-endian each), the expected 32-byte output and the
vector's name. Usage: make_bn254_pairing_golden.py [reference tests directory]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/tests"


def main():
    with open(os.path.join(REF, "protocol_ethereum_evm_precompiles", "bn256Pairing.json")) as f:
        src = json.load(f)
    vectors = [{"name": v["Name"], "input": v["Input"].lower(), "expected": v["Expected"].lower()} for v in src]
    for v in vectors:
        assert len(v["input"]) % 384 == 0 and len(v["expected"]) == 64
    out = {"source": "reference tests/protocol_ethereum_evm_precompiles/bn256Pairing.json", "vectors": vectors}
    with open(os.path.join(HERE, "evm_bn254_pairing_kat.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote %d vectors" % len(vectors))


if __name__ == "__main__":
    main()
