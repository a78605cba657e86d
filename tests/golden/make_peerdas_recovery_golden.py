#!/usr/bin/env python3
"""Extract the reference's EIP-7594 recover_cells_and_kzg_proofs known answers.

Source (dev container only):
  reference tests/protocol_ethereum_eip7594_fulu_peerdas/recover_cells_and_kzg_proofs/kzg-mainnet/*/data.yaml
  (cell_indices + cells -> [cells, proofs] or null)
Every input cell that is a cell of one of the seven blobs of tests/golden/kzg_commit_kat.npz is stored as [blob, cell]; the others (the
deliberately corrupted cells and the cells of the wrong length) are stored as hex. A valid case's output is stored as the index of its
source blob: tests/golden/peerdas_kat.npz already holds that blob's cell digests and proofs. Before anything is written:
  - the exact tier (tests/peerdas_recovery_exact.py, recover_polynomial) reproduces every cell of every valid output;
  - every valid output equals the cell digests and proofs that peerdas_kat.npz holds for the source blob.
Output: tests/golden/peerdas_recovery_kat.npz
"""
import glob
import hashlib
import json
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kzg_exact as K  # noqa: E402
import peerdas_exact as P  # noqa: E402
import peerdas_recovery_exact as RX  # noqa: E402

REF = "/root/reference/tests/protocol_ethereum_eip7594_fulu_peerdas/recover_cells_and_kzg_proofs/kzg-mainnet"
LENGTHS, NOT_ASCENDING, SCALAR_LARGER = 2, 9, 4   # cttEthKzg_InputsLengthsMismatch, _CellIndicesNotAscending, _ScalarLargerThanCurveOrder


def case(path):
    y = open(os.path.join(path, "data.yaml")).read()
    inp, out = re.search(r"input:(.*)output:(.*)", y, re.S).groups()
    idx = [int(v) for v in re.findall(r"\d+", re.search(r"cell_indices: \[(.*?)\]", inp, re.S).group(1))]
    cells = [bytes.fromhex(h) for h in re.findall(r"'0x([0-9a-f]*)'", inp)]
    out = out.strip()
    if out.startswith("null"):
        return idx, cells, None, None
    hexes = re.findall(r"'0x([0-9a-f]*)'", out)
    rc = [bytes.fromhex(h) for h in hexes if len(h) == 2 * P.BYTES_PER_CELL]
    rp = [bytes.fromhex(h) for h in hexes if len(h) == 96]
    assert len(rc) == P.CELLS and len(rp) == P.CELLS
    return idx, cells, rc, rp


def outcome(idx, cells):
    """The reference's checks in order; "length" where the Python wrapper refuses the input before the C call."""
    if len(idx) != len(cells) or any(len(c) != P.BYTES_PER_CELL for c in cells):
        return "length", "unequal numbers of indices and cells, or a cell that is not 2048 bytes (Python wrapper: ValueError)"
    if not P.CELLS // 2 <= len(cells) <= P.CELLS:
        return LENGTHS, f"{len(cells)} cells: fewer than 64 or more than 128 -> cttEthKzg_InputsLengthsMismatch"
    if any(i >= P.CELLS for i in idx):
        return LENGTHS, "an index >= 128 (checked over all indices before the order) -> cttEthKzg_InputsLengthsMismatch"
    if any(a >= b for a, b in zip(idx, idx[1:])):
        return NOT_ASCENDING, "indices not strictly ascending -> cttEthKzg_CellIndicesNotAscending"
    if any(v >= K.R for c in cells for v in RX.cell_values(c)):
        return SCALAR_LARGER, "an element >= r: cellToCosetEvals -> cttEthKzg_ScalarLargerThanCurveOrder"
    raise AssertionError("a valid input among the invalid cases")


def main():
    blobs = [bytes(b) for b in np.load(os.path.join(HERE, "kzg_commit_kat.npz"))["blobs"]]
    das = json.loads(str(np.load(os.path.join(HERE, "peerdas_kat.npz"))["cases"]))
    known = {v["blob"]: v for v in das["compute_cells_and_kzg_proofs"]["valid"]}
    assert sorted(known) == list(range(len(blobs)))
    where = {}
    for j, b in enumerate(blobs):
        for k, c in enumerate(P.compute_cells(b)):
            where.setdefault(c, [j, k])

    def ref(c):
        return where.get(c, c.hex())

    valid, invalid = [], []
    for d in sorted(glob.glob(f"{REF}/*")):
        name = os.path.basename(d)
        idx, cells, rc, rp = case(d)
        rec = {"name": name, "cell_indices": idx, "cells": [ref(c) for c in cells]}
        if rc is None:
            rec["outcome"], rec["note"] = outcome(idx, cells)
            invalid.append(rec)
            continue
        coefs = RX.recover_polynomial(idx, [RX.cell_values(c) for c in cells])
        assert [P.cell_bytes(c) for c in RX.recovered_cells(coefs)] == rc, name
        src = [j for j, v in known.items() if v["cell_sha256"] == [hashlib.sha256(c).hexdigest() for c in rc]]
        assert src and known[src[0]]["proofs"] == [p.hex() for p in rp], name
        rec["blob"] = src[0]
        valid.append(rec)
    assert (len(valid), len(invalid)) == (4, 14)
    np.savez_compressed(os.path.join(HERE, "peerdas_recovery_kat.npz"), cases=np.array(json.dumps({"valid": valid, "invalid": invalid})))
    for c in invalid:
        print(c["name"], c["outcome"], c["note"])
    print("wrote peerdas_recovery_kat.npz", os.path.getsize(os.path.join(HERE, "peerdas_recovery_kat.npz")), "bytes")


if __name__ == "__main__":
    main()
