#!/usr/bin/env python3
"""EIP-4844 entries on the resident setup: commitments and blob proofs, n single calls against one batched call, with and without
the window table, and the split of one proof call (host checks + SHA-256, k_kzg_* kernels, MSM). The PeerDAS leg: the one-time
load_peerdas, compute_cells_and_kzg_proofs as n single calls against one batched call, and the split of a call (host, Fr kernels,
bank MSM with its engine phases, EC FFTs). The recovery leg: recover_cells_and_kzg_proofs with 64 seeded random cells missing per
blob, as n single calls against one batched call, and the same split. Prints one JSON line.
python tools/bench_kzg.py [--reps R] [--sizes 1,6,9,32,128] [--das-sizes 1,6,21,72] [--rec-sizes 1,6,21,72]"""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import bench  # noqa: E402
from constantine_b200 import msm as M  # noqa: E402


def random_blobs(n, seed):
    """n blobs of canonical field elements (top byte < 0x73 keeps every element below r)."""
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 256, size=(n, 4096, 32), dtype=np.uint8)
    b[:, :, 0] %= 0x73
    return [bytes(x) for x in b.reshape(n, -1)]


def timed(fn, reps):
    fn()
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(ts), 3)


def peerdas(ctx, sizes, reps):
    mono = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_kat.npz"))["srs_monomial_compressed"].tobytes()
    r = {}
    t0 = time.perf_counter()
    ctx.load_peerdas(mono)
    r["load_peerdas_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    blobs = random_blobs(max(sizes), 7594)
    for n in sizes:
        bs = blobs[:n]
        r[f"cells_proofs_single_x{n}_ms"] = timed(lambda: [ctx.compute_cells_and_kzg_proofs(b) for b in bs], reps)
        r[f"cells_proofs_batched_n{n}_ms"] = timed(lambda: ctx.compute_cells_and_kzg_proofs_batch(bs), reps)
        splits = []
        for _ in range(reps):
            t0 = time.perf_counter()
            ctx.compute_cells_and_kzg_proofs_batch(bs)
            wall = (time.perf_counter() - t0) * 1e3
            st = M.last_stats()
            splits.append({"wall_ms": wall, **ctx.last_das_timing(), **{k: st[k] for k in ("ms_digits", "ms_sort", "ms_accumulate",
                                                                                          "ms_fixup", "ms_reduce", "ms_d2h_tail")}})
        r[f"split_n{n}_ms"] = {k: round(statistics.median(s[k] for s in splits), 3) for k in splits[0]}
        r[f"msm_c_n{n}"] = M.last_stats()["c"]
    r["cells_only_x1_ms"] = timed(lambda: ctx.compute_cells(blobs[0]), reps)
    return r


def recovery(ctx, sizes, reps):
    """Needs load_peerdas (the PeerDAS leg runs first). Each blob keeps 64 of its 128 cells, chosen by a seeded generator."""
    blobs = random_blobs(max(sizes), 7596)
    rnd = random.Random(7596)
    items = []
    for cells, _ in ctx.compute_cells_and_kzg_proofs_batch(blobs):
        idx = sorted(rnd.sample(range(128), 64))
        items.append((idx, [cells[i] for i in idx]))
    r = {}
    for n in sizes:
        its = items[:n]
        r[f"recover_single_x{n}_ms"] = timed(lambda: [ctx.recover_cells_and_kzg_proofs(i, c) for i, c in its], reps)
        r[f"recover_batched_n{n}_ms"] = timed(lambda: ctx.recover_cells_and_kzg_proofs_batch(its), reps)
        splits = []
        for _ in range(reps):
            t0 = time.perf_counter()
            ctx.recover_cells_and_kzg_proofs_batch(its)
            splits.append({"wall_ms": (time.perf_counter() - t0) * 1e3, **ctx.last_das_timing()})
        r[f"split_n{n}_ms"] = {k: round(statistics.median(s[k] for s in splits), 3) for k in splits[0]}
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1,6,9,32,128")
    ap.add_argument("--das-sizes", default="1,6,21,72")
    ap.add_argument("--rec-sizes", default="1,6,21,72")
    a = ap.parse_args()
    sizes = [int(s) for s in a.sizes.split(",")]
    srs = np.load(os.path.join(ROOT, "tests", "golden", "kzg_commit_kat.npz"))["srs_lagrange_brp_compressed"].tobytes()
    ctx = M.EthKzgContext(srs, compressed=True)
    blobs = random_blobs(max(sizes), 4844)
    cms = ctx.blobs_to_kzg_commitments(blobs)
    out = {"gpu": bench.gpu_identity(0), "reps": a.reps, "modes": {}}
    for mode in ("plain", "table"):
        r = {}
        if mode == "table":
            r["c"] = ctx.precompute(0)
        for n in sizes:
            bs, cs = blobs[:n], cms[:n]
            r[f"commit_single_x{n}_ms"] = timed(lambda: [ctx.blob_to_kzg_commitment(b) for b in bs], a.reps)
            r[f"commit_batched_n{n}_ms"] = timed(lambda: ctx.blobs_to_kzg_commitments(bs), a.reps)
            r[f"blob_proof_single_x{n}_ms"] = timed(lambda: [ctx.compute_blob_kzg_proof(b, c) for b, c in zip(bs, cs)], a.reps)
            r[f"blob_proof_batched_n{n}_ms"] = timed(lambda: ctx.compute_blob_kzg_proofs(bs, cs), a.reps)
        # split of one proof call: host checks + challenge, the quotient kernels (events), the MSM (engine phase timer)
        splits = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            ctx.compute_blob_kzg_proof(blobs[0], cms[0])
            wall = (time.perf_counter() - t0) * 1e3
            splits.append({"wall_ms": wall, **ctx.last_timing(), "ms_msm": M.last_stats()["ms_total"]})
        r["blob_proof_split_ms"] = {k: round(statistics.median(s[k] for s in splits), 3) for k in splits[0]}
        out["modes"][mode] = r
    out["peerdas"] = peerdas(ctx, [int(s) for s in a.das_sizes.split(",")], a.reps)
    out["recovery"] = recovery(ctx, [int(s) for s in a.rec_sizes.split(",")], a.reps)
    ctx.delete()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
