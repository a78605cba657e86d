#!/usr/bin/env python3
"""Build tests/golden/evm_curve_ops_kat.json from the reference's vectors of the EVM curve additions and scalar multiplications
(run where the reference tree exists; the fixture -- not this script -- is what the tests read).

Sources (reference tests/protocol_ethereum_evm_precompiles/): bn256Add.json (ECADD), bn256ScalarMul.json (ECMUL),
eip-2537/{,fail-}{add,mul}_G{1,2}_bls.json and blsG1AddNimbus.json (BLS12_G1ADD). Per precompile, a list of vectors: the name, the
hex input, and either the expected output (status cttEVM_Success) or the status its "ExpectedError" string maps to (ERRORS).
Usage: make_evm_curve_ops_golden.py [reference tests directory]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/tests"

# substrings of the error strings -> ctt_evm_status names
ERRORS = (("invalid input length", "cttEVM_InvalidInputSize"),
          ("top bytes", "cttEVM_IntLargerThanModulus"),
          ("encoding", "cttEVM_IntLargerThanModulus"),
          ("modulus", "cttEVM_IntLargerThanModulus"),
          ("not on curve", "cttEVM_PointNotOnCurve"),
          ("not on correct subgroup", "cttEVM_PointNotInSubgroup"))


def status_of(err):
    hits = [st for key, st in ERRORS if key in err]
    assert len(hits) == 1, err
    return hits[0]


def load(name):
    with open(os.path.join(REF, "protocol_ethereum_evm_precompiles", name + ".json")) as f:
        return json.load(f)


def vectors(name):
    out = []
    for v in load(name):
        if v.get("ExpectedError"):
            out.append({"name": v["Name"], "input": v["Input"].lower(), "status": status_of(v["ExpectedError"]), "expected": ""})
        else:
            out.append({"name": v["Name"], "input": v["Input"].lower(), "status": "cttEVM_Success", "expected": v["Expected"].lower()})
    return out


def main():
    out = {"source": "reference tests/protocol_ethereum_evm_precompiles: bn256Add.json, bn256ScalarMul.json, "
                     "eip-2537/{,fail-}{add,mul}_G{1,2}_bls.json, blsG1AddNimbus.json"}
    out["bn254_g1add"] = vectors("bn256Add")
    out["bn254_g1mul"] = vectors("bn256ScalarMul")
    for op, stem in (("bls12381_g1add", "add_G1"), ("bls12381_g2add", "add_G2"), ("bls12381_g1mul", "mul_G1"),
                     ("bls12381_g2mul", "mul_G2")):
        out[op] = vectors("eip-2537/%s_bls" % stem) + vectors("eip-2537/fail-%s_bls" % stem)
    out["bls12381_g1add"] += vectors("blsG1AddNimbus")
    counts = {k: len(v) for k, v in out.items() if isinstance(v, list)}
    assert counts == {"bn254_g1add": 16, "bn254_g1mul": 19, "bls12381_g1add": 9 + 6 + 110, "bls12381_g2add": 9 + 6,
                      "bls12381_g1mul": 11 + 7, "bls12381_g2mul": 11 + 7}, counts
    with open(os.path.join(HERE, "evm_curve_ops_kat.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote %s" % counts)


if __name__ == "__main__":
    main()
