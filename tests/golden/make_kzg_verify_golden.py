#!/usr/bin/env python3
"""Extract the reference's EIP-4844 verify_kzg_proof, verify_blob_kzg_proof and verify_blob_kzg_proof_batch known answers.

Sources (dev container only):
  reference tests/protocol_ethereum_eip4844_deneb_kzg/verify_kzg_proof/kzg-mainnet/*/data.yaml             (commitment, z, y, proof)
  reference tests/protocol_ethereum_eip4844_deneb_kzg/verify_blob_kzg_proof/kzg-mainnet/*/data.yaml        (blob, commitment, proof)
  reference tests/protocol_ethereum_eip4844_deneb_kzg/verify_blob_kzg_proof_batch/kzg-mainnet/*/data.yaml  (blobs, commitments, proofs)
each -> true / false / null. Every full-length blob is one of the seven blobs of tests/golden/kzg_commit_kat.npz (stored as
["valid", index]) or one of the two bad blobs of tests/golden/kzg_proof_kat.npz (["bad", index]); the two others have the wrong length
(["length", bytes]). A null case's outcome is the exact status, found by walking the reference's check order
(tests/kzg_verify_exact.py, status_*) with the point statuses of make_kzg_proof_golden.commitment_status; lists of unequal length and
items of the wrong size are "length" (fixed-size C arguments cannot express them: the Python methods refuse them before the call).
The G2 setup is that of tests/golden/peerdas_verify_kat.npz. The counts of the three entries are asserted before anything is written.
Output: tests/golden/kzg_verify_kat.npz
"""
import glob
import json
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
import kzg_exact as K  # noqa: E402
import kzg_verify_exact as VE  # noqa: E402
import make_kzg_proof_golden as KG  # noqa: E402

REF = "/root/reference/tests/protocol_ethereum_eip4844_deneb_kzg"


def one(y, key):
    return bytes.fromhex(re.search(key + r": '0x([0-9a-f]*)'", y).group(1))


def many(y, key):
    return [bytes.fromhex(h) for h in re.findall(r"'0x([0-9a-f]*)'", re.search(key + r": \[(.*?)\]", y, re.S).group(1))]


def result(y):
    o = re.search(r"output: (.*)", y, re.S).group(1).strip()
    return None if o.startswith("null") else o.startswith("true")


def point_status(b):
    return KG.commitment_status(b)[0]


def main():
    blobs = [bytes(b) for b in np.load(os.path.join(HERE, "kzg_commit_kat.npz"))["blobs"]]
    bad = [bytes(b) for b in np.load(os.path.join(HERE, "kzg_proof_kat.npz"))["bad_blobs"]]

    def blob_ref(b):
        if len(b) != K.BYTES_PER_BLOB:
            return ["length", len(b)]
        if b in blobs:
            return ["valid", blobs.index(b)]
        return ["bad", bad.index(b)]                     # raises for an unknown blob

    def outcome(res, sized, status):
        if res is not None:
            return VE.SUCCESS if res else VE.FAILURE
        if not sized:
            return "length"
        st = status()
        assert st not in (VE.SUCCESS, VE.FAILURE)
        return st

    cases = {"verify_kzg_proof": [], "verify_blob_kzg_proof": [], "verify_blob_kzg_proof_batch": []}
    for d in sorted(glob.glob(f"{REF}/verify_kzg_proof/kzg-mainnet/*")):
        y = open(os.path.join(d, "data.yaml")).read()
        c, z, v, p = one(y, "commitment"), one(y, "z"), one(y, "y"), one(y, "proof")
        sized = (len(c), len(z), len(v), len(p)) == (48, 32, 32, 48)
        cases["verify_kzg_proof"].append({
            "name": os.path.basename(d), "commitment": c.hex(), "z": z.hex(), "y": v.hex(), "proof": p.hex(),
            "outcome": outcome(result(y), sized, lambda: VE.status_kzg_proof(c, z, v, p, point_status))})
    for d in sorted(glob.glob(f"{REF}/verify_blob_kzg_proof/kzg-mainnet/*")):
        y = open(os.path.join(d, "data.yaml")).read()
        b, c, p = one(y, "blob"), one(y, "commitment"), one(y, "proof")
        sized = (len(b), len(c), len(p)) == (K.BYTES_PER_BLOB, 48, 48)
        cases["verify_blob_kzg_proof"].append({
            "name": os.path.basename(d), "blob": blob_ref(b), "commitment": c.hex(), "proof": p.hex(),
            "outcome": outcome(result(y), sized, lambda: VE.status_blob_proof(b, c, p, point_status))})
    for d in sorted(glob.glob(f"{REF}/verify_blob_kzg_proof_batch/kzg-mainnet/*")):
        y = open(os.path.join(d, "data.yaml")).read()
        bs, cs, ps = many(y, "blobs"), many(y, "commitments"), many(y, "proofs")
        sized = (len(bs) == len(cs) == len(ps) and all(len(b) == K.BYTES_PER_BLOB for b in bs)
                 and all(len(x) == 48 for x in cs + ps))
        cases["verify_blob_kzg_proof_batch"].append({
            "name": os.path.basename(d), "blobs": [blob_ref(b) for b in bs], "commitments": [c.hex() for c in cs],
            "proofs": [p.hex() for p in ps],
            "outcome": outcome(result(y), sized, lambda: VE.status_blob_batch(bs, cs, ps, point_status))})

    counts = {k: (len(v), sum(c["outcome"] == 0 for c in v), sum(c["outcome"] == 1 for c in v)) for k, v in cases.items()}
    assert counts == {"verify_kzg_proof": (122, 54, 48), "verify_blob_kzg_proof": (29, 9, 8),
                      "verify_blob_kzg_proof_batch": (24, 7, 2)}, counts
    g2 = np.load(os.path.join(HERE, "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"]
    assert g2.size == 65 * 96
    np.savez_compressed(os.path.join(HERE, "kzg_verify_kat.npz"), cases=np.array(json.dumps(cases)))
    for k, v in cases.items():
        for c in v:
            if c["outcome"] not in (0, 1):
                print(k, c["name"], c["outcome"])
    print("wrote kzg_verify_kat.npz", os.path.getsize(os.path.join(HERE, "kzg_verify_kat.npz")), "bytes")


if __name__ == "__main__":
    main()
