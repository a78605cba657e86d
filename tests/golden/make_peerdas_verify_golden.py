#!/usr/bin/env python3
"""Extract the reference's EIP-7594 verify_cell_kzg_proof_batch known answers, its challenge vectors and the G2 trusted setup.

Source (dev container only):
  reference tests/protocol_ethereum_eip7594_fulu_peerdas/verify_cell_kzg_proof_batch/kzg-mainnet/*/data.yaml
    (commitments, cell_indices, cells, proofs -> true / false / null)
  reference tests/protocol_ethereum_eip7594_fulu_peerdas/compute_verify_cell_kzg_proof_batch_challenge/kzg-mainnet/*/data.yaml
    (commitments, commitment_indices, cell_indices, cosets_evals, proofs -> r)
  reference constantine/commitments_setups/trusted_setup_ethereum_kzg4844_reference.dat (the 65 monomial G2 points)
Every cell that is a cell of one of the seven blobs of tests/golden/kzg_commit_kat.npz is stored as [blob, cell]; the others as hex.
An error vector's outcome is the exact status, found by walking the reference's check order (tests/peerdas_verify_exact.py, status)
with the point statuses of make_kzg_proof_golden.commitment_status; the four length mismatches and the six items of the wrong size are
"length" (one num_cells and fixed-size items cannot express them: the Python method refuses them before the C call).
Before anything is written, the exact tier reproduces all 10 challenges.
Output: tests/golden/peerdas_verify_kat.npz
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
import make_kzg_proof_golden as KG  # noqa: E402
import peerdas_exact as P  # noqa: E402
import peerdas_verify_exact as VX  # noqa: E402

BASE = "/root/reference/tests/protocol_ethereum_eip7594_fulu_peerdas"
SETUP = "/root/reference/constantine/commitments_setups/trusted_setup_ethereum_kzg4844_reference.dat"


def hexes(block):
    return [bytes.fromhex(h) for h in re.findall(r"'0x([0-9a-f]*)'", block)]


def field(inp, key, nxt):
    m = re.search(key + r":(.*?)(?:\n  " + nxt + r":|\Z)", inp, re.S)
    return m.group(1)


def ints(inp, key):
    return [int(v) for v in re.findall(r"\d+", re.search(key + r": \[(.*?)\]", inp, re.S).group(1))]


def verify_case(path):
    y = open(os.path.join(path, "data.yaml")).read()
    inp, out = re.search(r"input:(.*)output:(.*)", y, re.S).groups()
    commitments = hexes(field(inp, "commitments", "cell_indices"))
    cells = hexes(field(inp, "cells", "proofs"))
    proofs = hexes(field(inp, "proofs", "ZZZ"))
    out = out.strip()
    res = None if out.startswith("null") else out.startswith("true")
    return commitments, ints(inp, "cell_indices"), cells, proofs, res


def challenge_case(path):
    y = open(os.path.join(path, "data.yaml")).read()
    inp, out = re.search(r"input:(.*)output:(.*)", y, re.S).groups()
    commitments = hexes(field(inp, "commitments", "commitment_indices"))
    evals = field(inp, "cosets_evals", "proofs")
    cells = [b"".join(hexes(c)) for c in re.split(r"\n  - - ", evals)[1:]] if "- - " in evals else []
    proofs = hexes(field(inp, "proofs", "ZZZ"))
    return commitments, ints(inp, "commitment_indices"), ints(inp, "cell_indices"), cells, proofs, hexes(out)[0]


def sized(commitments, cells, proofs):
    return all(len(c) == 48 for c in commitments + proofs) and all(len(c) == P.BYTES_PER_CELL for c in cells)


def main():
    blobs = [bytes(b) for b in np.load(os.path.join(HERE, "kzg_commit_kat.npz"))["blobs"]]
    where = {}
    for j, b in enumerate(blobs):
        for k, c in enumerate(P.compute_cells(b)):
            where.setdefault(c, [j, k])

    def ref(c):
        return where.get(c, c.hex())

    def point_status(b):
        return KG.commitment_status(b)[0]

    cases = []
    for d in sorted(glob.glob(f"{BASE}/verify_cell_kzg_proof_batch/kzg-mainnet/*")):
        name = os.path.basename(d)
        commitments, idx, cells, proofs, res = verify_case(d)
        rec = {"name": name, "commitments": [c.hex() for c in commitments], "cell_indices": idx, "cells": [ref(c) for c in cells],
               "proofs": [p.hex() for p in proofs]}
        if res is not None:
            assert len({len(commitments), len(idx), len(cells), len(proofs)}) == 1, name
            rec["outcome"] = VX.SUCCESS if res else VX.FAILURE
        elif len({len(commitments), len(idx), len(cells), len(proofs)}) != 1 or not sized(commitments, cells, proofs):
            rec["outcome"] = "length"
        else:
            rec["outcome"] = VX.status(commitments, idx, cells, proofs, point_status)
            assert rec["outcome"] not in (VX.SUCCESS, VX.FAILURE), name
        cases.append(rec)
    outcomes = [c["outcome"] for c in cases]
    assert (outcomes.count(0), outcomes.count(1), len(cases)) == (12, 3, 32), outcomes
    assert outcomes.count("length") == 10      # 4 unequal list lengths, 6 items of the wrong size

    challenges = []
    for d in sorted(glob.glob(f"{BASE}/compute_verify_cell_kzg_proof_batch_challenge/kzg-mainnet/*")):
        commitments, cidx, idx, cells, proofs, out = challenge_case(d)
        assert len(cidx) == len(idx) == len(cells) == len(proofs), d
        assert VX.challenge(commitments, cidx, idx, cells, proofs) == int.from_bytes(out, "big"), d
        challenges.append({"name": os.path.basename(d), "commitments": [c.hex() for c in commitments], "commitment_indices": cidx,
                           "cell_indices": idx, "cells": [ref(c) for c in cells], "proofs": [p.hex() for p in proofs], "challenge": out.hex()})
    assert len(challenges) == 10

    words = open(SETUP).read().split()
    n1, n2 = int(words[0]), int(words[1])
    g2 = words[2 + n1:2 + n1 + n2]
    assert (n1, n2) == (4096, 65) and all(len(h) == 192 for h in g2)
    np.savez_compressed(os.path.join(HERE, "peerdas_verify_kat.npz"),
                        cases=np.array(json.dumps({"verify": cases, "challenge": challenges})),
                        srs_monomial_g2_compressed=np.frombuffer(bytes.fromhex("".join(g2)), dtype=np.uint8))
    for c in cases:
        print(c["name"], c["outcome"])
    print("wrote peerdas_verify_kat.npz", os.path.getsize(os.path.join(HERE, "peerdas_verify_kat.npz")), "bytes")


if __name__ == "__main__":
    main()
