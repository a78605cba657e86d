#!/usr/bin/env python3
"""Write tests/golden/bls_kat.json: the Ethereum BLS signature vectors the suite checks.

  python tests/golden/make_bls_golden.py <constantine checkout>

Sources (inside the checkout):
  tests/protocol_hash_to_curve/tv_h2c_v8_BLS12_381_hash_to_G2_SHA256_SSWU_RO.json       the 5 RFC 9380 hash_to_G2 vectors
  tests/protocol_blssig_pop_on_bls12381_g2_test_vectors_v0.1.1/<kind>/*.json           the Ethereum vectors
  include/constantine/protocols/ethereum_bls_signatures.h, ..._parallel.h             the prototypes of the verification symbols

Deserialization vectors get the exact ctt_codec_ecc_status the reference's deserialize_g1_compressed / deserialize_g2_compressed
(constantine/serialization/codecs_bls12_381.nim) return, computed here by the same steps in the same order: the compressed flag and
the infinity encoding (1), infinity itself (5, PointAtInfinity, not Success), x >= p (2; for G2 x.c1 first, then x.c0), not on the
curve (3), not in the subgroup (4), else 0. Inputs of the wrong length have no status (the C entries take fixed-size arrays): "length".
"""
import glob
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "tools"))
import gen_bls_constants as G  # noqa: E402

P, R = G.P, G.R
COUNTS = {"hash_to_G2": 4, "verify": 29, "aggregate_verify": 5, "fast_aggregate_verify": 12, "batch_verify": 2,
          "deserialization_G1": 13, "deserialization_G2": 15}


# ---- minimal affine arithmetic for the subgroup checks (Fp as degenerate Fp2 for G1) ----------------------------------------
def ec_add(p1, p2):
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    (x1, y1), (x2, y2) = p1, p2
    if x1 == x2:
        if G.add(y1, y2) == G.ZERO:
            return None
        lam = G.mul(G.smul(3, G.mul(x1, x1)), G.inv(G.smul(2, y1)))
    else:
        lam = G.mul(G.sub(y2, y1), G.inv(G.sub(x2, x1)))
    x3 = G.sub(G.sub(G.mul(lam, lam), x1), x2)
    return x3, G.sub(G.mul(lam, G.sub(x1, x3)), y1)


def ec_mul(k, pt):
    acc = None
    for bit in bin(k)[2:]:
        acc = ec_add(acc, acc)
        if bit == "1":
            acc = ec_add(acc, pt)
    return acc


def decode_status(raw, g2):
    size = 96 if g2 else 48
    if len(raw) != size:
        return "length"
    if not raw[0] & 0x80:
        return 1
    if raw[0] & 0x40:
        if raw[0] & 0x3F or any(raw[1:]):
            return 1
        return 5
    c1 = int.from_bytes(raw[:48], "big") & ((1 << 381) - 1)
    if c1 >= P:
        return 2
    if g2:
        c0 = int.from_bytes(raw[48:], "big")
        if c0 >= P:
            return 2
        x, b = (c0, c1), G.B_E2
    else:
        x, b = (c1, 0), (4, 0)
    y = G.sqrt(G.add(G.mul(G.mul(x, x), x), b))
    if y is None or (not g2 and y[1] != 0):
        return 3
    return 0 if ec_mul(R, (x, y)) is None else 4


def prototypes(ref):
    out = {}
    for hdr in ("ethereum_bls_signatures.h", "ethereum_bls_signatures_parallel.h"):
        text = open(os.path.join(ref, "include", "constantine", "protocols", hdr)).read()
        for name in ("ctt_eth_bls_batch_verify_parallel", "ctt_eth_bls_batch_verify", "ctt_eth_bls_aggregate_verify"):
            m = re.search(r"ctt_eth_bls_status\s+%s\s*\(([^;]*?)\)\s*__attribute__" % name, text, re.S)
            if m and name not in out:
                out[name] = " ".join(m.group(1).split())
    assert sorted(out) == sorted(["ctt_eth_bls_batch_verify_parallel", "ctt_eth_bls_batch_verify", "ctt_eth_bls_aggregate_verify"]), out
    return out


def main(ref):
    h2c = json.load(open(os.path.join(ref, "tests", "protocol_hash_to_curve", "tv_h2c_v8_BLS12_381_hash_to_G2_SHA256_SSWU_RO.json")))
    vecs = [{"msg": v["msg"], "u0": v["u"][0], "u1": v["u"][1], "Q0": v["Q0"], "Q1": v["Q1"], "P": v["P"]} for v in h2c["vectors"]]
    assert len(vecs) == 5
    out = {"rfc_h2c": {"dst": h2c["dst"], "vectors": vecs}}
    base = os.path.join(ref, "tests", "protocol_blssig_pop_on_bls12381_g2_test_vectors_v0.1.1")
    for kind, count in COUNTS.items():
        items = []
        for path in sorted(glob.glob(os.path.join(base, kind, "*.json"))):
            d = json.load(open(path))
            d["name"] = os.path.basename(path)[:-5]
            if kind.startswith("deserialization"):
                key = "pubkey" if kind.endswith("G1") else "signature"
                d["status"] = decode_status(bytes.fromhex(d["input"][key]), kind.endswith("G2"))
                assert (d["status"] == 0 or d["status"] == 5) == d["output"], (path, d["status"])
            items.append(d)
        assert len(items) == count, (kind, len(items))
        out[kind] = items
    out["prototypes"] = prototypes(ref)
    with open(os.path.join(HERE, "bls_kat.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote bls_kat.json:", {k: len(v) for k, v in out.items() if isinstance(v, list)})


if __name__ == "__main__":
    main(sys.argv[1])
