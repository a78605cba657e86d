"""Regenerates tests/golden/divstep_worst.json: for every field of constantine_b200/curves.py, the 256 inputs in [1, p) with the
most half-delta divsteps (the count the safegcd inversion of field_inv.cuh runs before g reaches zero), found among 2^20 seeded
uniform candidates. tests/test_arith_edges.py recounts them, feeds them to the device inversions and checks the batch bound.

    python tests/golden/make_divstep_golden.py      # ~10 min on 8 cores
"""
import heapq
import json
import os
import random
import sys
from multiprocessing import Pool

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from constantine_b200.curves import FIELDS  # noqa: E402

CANDIDATES = 1 << 20
KEEP = 256
CHUNKS = 64


def divsteps(p, x):
    """Half-delta divsteps from (delta, f, g) = (1/2, p, x) until g = 0; zeta = -(delta + 1/2) as in field_inv.cuh."""
    f, g, zeta, n = p, x, -1, 0
    while g:
        if not g & 1:
            t = (g & -g).bit_length() - 1          # a run of even steps: g / 2, delta + 1 each
            g >>= t
            zeta -= t
            n += t
            continue
        if zeta < 0:
            f, g, zeta = g, (g - f) >> 1, -zeta - 2
        else:
            g, zeta = (g + f) >> 1, zeta - 1
        n += 1
    return n


def _chunk(args):
    name, k = args
    p = FIELDS[name].modulus
    rnd = random.Random("%s/%d" % (name, k))
    heap = []
    for _ in range(CANDIDATES // CHUNKS):
        x = rnd.randrange(1, p)
        item = (divsteps(p, x), x)
        if len(heap) < KEEP:
            heapq.heappush(heap, item)
        elif item > heap[0]:
            heapq.heapreplace(heap, item)
    return name, heap


def main():
    out = {"candidates_per_field": CANDIDATES, "fields": {}}
    best = {name: [] for name in FIELDS}
    with Pool() as pool:
        for name, heap in pool.imap_unordered(_chunk, [(n, k) for n in FIELDS for k in range(CHUNKS)]):
            best[name] = heapq.nlargest(KEEP, best[name] + heap)
    for name in FIELDS:
        out["fields"][name] = [[n, hex(x)] for n, x in best[name]]
    with open(os.path.join(ROOT, "tests", "golden", "divstep_worst.json"), "w") as f:
        json.dump(out, f, indent=0)
        f.write("\n")
    print({name: best[name][0][0] for name in FIELDS})


if __name__ == "__main__":
    main()
