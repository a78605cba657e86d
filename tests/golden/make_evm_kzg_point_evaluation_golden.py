#!/usr/bin/env python3
"""Build tests/golden/evm_kzg_point_evaluation_kat.json (the fixture, not this script, is what the tests read).

Source: the reference's tests/protocol_ethereum_evm_precompiles/eip-4844/pointEvaluation.json, geth's vector for the POINT_EVALUATION
precompile (0x0a): its Input, its Expected output and its name, kept as they are. The other cases of the tests come from the
verify_kzg_proof vectors already in tests/golden/kzg_verify_kat.npz. Usage: make_evm_kzg_point_evaluation_golden.py [reference tests
directory]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/tests"


def main():
    with open(os.path.join(REF, "protocol_ethereum_evm_precompiles", "eip-4844", "pointEvaluation.json")) as f:
        vs = json.load(f)
    out = {"source": "reference tests/protocol_ethereum_evm_precompiles/eip-4844/pointEvaluation.json (geth's vector)",
           "vectors": [{"name": v["Name"], "input": v["Input"], "expected": v["Expected"], "gas": v["Gas"]} for v in vs]}
    with open(os.path.join(HERE, "evm_kzg_point_evaluation_kat.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote %d vector(s)" % len(vs))


if __name__ == "__main__":
    main()
