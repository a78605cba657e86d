#!/usr/bin/env python3
"""Build tests/golden/eip2537_pairing_map_kat.json from the reference's EIP-2537 pairing-check and map vectors and the RFC 9380
hash-to-G1 vectors (run where the reference tree exists; the fixture -- not this script -- is what the tests and
tools/gen_bls_constants.py read).

Sources (reference tests/):
  - protocol_ethereum_evm_precompiles/eip-2537/{,fail-}pairing_check_bls.json, {,fail-}map_fp_to_G1_bls.json,
    {,fail-}map_fp2_to_G2_bls.json (the go-ethereum suite): per vector the hex input, the expected output (success files) or the
    expected ctt_evm_status (fail files, the error strings mapped by FAIL_STATUS of tests/eip2537_exact.py);
  - protocol_hash_to_curve/tv_h2c_v8_BLS12_381_hash_to_G1_SHA256_SSWU_RO.json: msg, u0, u1, Q0, Q1 (the SSWU-and-isogeny images of
    u0 and u1, before the cofactor clearing) and P = clear(Q0 + Q1), coordinates as hex strings.
Usage: make_eip2537_pairing_map_golden.py [reference tests directory]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.dont_write_bytecode = True
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/tests"

from eip2537_exact import FAIL_STATUS  # noqa: E402


def load(name):
    with open(os.path.join(REF, "protocol_ethereum_evm_precompiles", "eip-2537", name + ".json")) as f:
        return json.load(f)


def main():
    out = {"source": "reference tests/protocol_ethereum_evm_precompiles/eip-2537 and "
                     "tests/protocol_hash_to_curve/tv_h2c_v8_BLS12_381_hash_to_G1_SHA256_SSWU_RO.json"}
    for key, name in (("pairing", "pairing_check_bls"), ("map_g1", "map_fp_to_G1_bls"), ("map_g2", "map_fp2_to_G2_bls")):
        out[key] = [{"name": v["Name"], "input": v["Input"].lower(), "expected": v["Expected"].lower()} for v in load(name)]
        out[key + "_fail"] = [{"name": v["Name"], "input": v["Input"].lower(), "status": FAIL_STATUS[v["ExpectedError"]]}
                              for v in load("fail-" + name)]
    with open(os.path.join(REF, "protocol_hash_to_curve", "tv_h2c_v8_BLS12_381_hash_to_G1_SHA256_SSWU_RO.json")) as f:
        h2c = json.load(f)
    out["rfc_h2g1"] = {"dst": h2c["dst"], "vectors": [
        {"msg": v["msg"], "u0": v["u"][0], "u1": v["u"][1], "Q0": v["Q0"], "Q1": v["Q1"], "P": v["P"]} for v in h2c["vectors"]]}
    assert len(out["pairing"]) == 10 and len(out["pairing_fail"]) == 22 and len(out["rfc_h2g1"]["vectors"]) == 5
    with open(os.path.join(HERE, "eip2537_pairing_map_kat.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote %s" % {k: len(v) for k, v in out.items() if isinstance(v, list)})


if __name__ == "__main__":
    main()
