#!/usr/bin/env python3
"""EIP-4844 entries on the resident setup: commitments and blob proofs, n single calls against one batched call, with and without
the window table, and the split of one proof call (host checks + SHA-256, k_kzg_* kernels, MSM). The PeerDAS leg: the one-time
load_peerdas, compute_cells_and_kzg_proofs as n single calls against one batched call, and the split of a call (host, Fr kernels,
bank MSM with its engine phases, EC FFTs). The recovery leg: recover_cells_and_kzg_proofs with 64 seeded random cells missing per
blob, as n single calls against one batched call, and the same split. The verify leg: verify_cell_kzg_proof_batch over n cells of 72
random blobs (n = 128, 6 x 128, 21 x 128, 72 x 128 shuffled; one column of 72; 8 columns of 72), with the Fiat-Shamir challenge and with
caller-supplied random bytes: the median per call and its split (host checks + challenge, device decode, scalar kernels, bank MSM,
host pairing). The verify4844 leg: verify_blob_kzg_proof_batch over n seeded random blobs with their device-computed commitments and
proofs, with the Fiat-Shamir r and with caller-supplied random bytes, the same split, and the single entries verify_blob_kzg_proof and
verify_kzg_proof. Prints one JSON line.
python tools/bench_kzg.py [--reps R] [--sizes 1,6,9,32,128] [--das-sizes 1,6,21,72] [--rec-sizes 1,6,21,72] [--verify-sizes 1,6,21,72]
                          [--verify4844-sizes 1,6,72,1024] [--only verify|verify4844]"""
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


def verify(ctx, sizes, reps):
    """Needs load_peerdas (the PeerDAS leg or the caller loads it). sizes: numbers of 128-cell rows."""
    ctx.load_g2_setup(np.load(os.path.join(ROOT, "tests", "golden", "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes())
    blobs = random_blobs(72, 7597)
    cms = ctx.blobs_to_kzg_commitments(blobs)
    full = ctx.compute_cells_and_kzg_proofs_batch(blobs)
    rnd = random.Random(7597)
    every = [(b, c) for b in range(72) for c in range(128)]
    rnd.shuffle(every)
    shapes = {f"cells{128 * n}": every[:128 * n] for n in sizes}
    shapes["col1x72"] = [(b, 77) for b in range(72)]
    shapes["col8x72"] = [(b, c) for c in range(0, 128, 16) for b in range(72)]
    r = {}
    for name, picks in shapes.items():
        a = ([cms[b] for b, _ in picks], [c for _, c in picks], [full[b][0][c] for b, c in picks], [full[b][1][c] for b, c in picks])
        for path, rb in (("fs", bytes(32)), ("rand", bytes(range(1, 33)))):
            assert ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=rb)
            splits = []
            ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=rb)
            for _ in range(reps):
                t0 = time.perf_counter()
                ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=rb)
                splits.append({"wall_ms": (time.perf_counter() - t0) * 1e3, **ctx.last_verify_timing()})
            r[f"{name}_{path}_ms"] = {k: round(statistics.median(s[k] for s in splits), 3) for k in splits[0]}
    return r


def verify4844(ctx, sizes, reps):
    """verify_blob_kzg_proof_batch over n blobs (both r paths) and the single entries; needs only the G2 setup."""
    ctx.load_g2_setup(np.load(os.path.join(ROOT, "tests", "golden", "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes())
    blobs = random_blobs(max(sizes), 4845)
    cms = ctx.blobs_to_kzg_commitments(blobs)
    proofs = ctx.compute_blob_kzg_proofs(blobs, cms)
    r = {}

    def split(fn):
        assert fn()
        fn()
        s = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            s.append({"wall_ms": (time.perf_counter() - t0) * 1e3, **ctx.last_verify_timing()})
        return {k: round(statistics.median(x[k] for x in s), 3) for k in s[0]}
    for n in sizes:
        a = (blobs[:n], cms[:n], proofs[:n])
        for path, rb in (("fs", bytes(32)), ("rand", bytes(range(1, 33)))):
            r[f"batch_n{n}_{path}_ms"] = split(lambda: ctx.verify_blob_kzg_proof_batch(*a, secure_random_bytes=rb))
    r["blob_proof_single_ms"] = split(lambda: ctx.verify_blob_kzg_proof(blobs[0], cms[0], proofs[0]))
    z = (4844).to_bytes(32, "big")
    proof, y = ctx.compute_kzg_proof(blobs[0], z)
    r["kzg_proof_single_ms"] = split(lambda: ctx.verify_kzg_proof(cms[0], z, y, proof))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1,6,9,32,128")
    ap.add_argument("--das-sizes", default="1,6,21,72")
    ap.add_argument("--rec-sizes", default="1,6,21,72")
    ap.add_argument("--verify-sizes", default="1,6,21,72")
    ap.add_argument("--verify4844-sizes", default="1,6,72,1024")
    ap.add_argument("--only", default="", help="'verify': only the verify leg (after load_peerdas); 'verify4844': only the verify4844 leg")
    a = ap.parse_args()
    sizes = [int(s) for s in a.sizes.split(",")]
    srs = np.load(os.path.join(ROOT, "tests", "golden", "kzg_commit_kat.npz"))["srs_lagrange_brp_compressed"].tobytes()
    ctx = M.EthKzgContext(srs, compressed=True)
    vsizes = [int(s) for s in a.verify_sizes.split(",")]
    v4sizes = [int(s) for s in a.verify4844_sizes.split(",")]
    if a.only == "verify4844":
        print(json.dumps({"gpu": bench.gpu_identity(0), "reps": a.reps, "verify4844": verify4844(ctx, v4sizes, a.reps)}), flush=True)
        ctx.delete()
        return
    if a.only == "verify":
        ctx.load_peerdas(np.load(os.path.join(ROOT, "tests", "golden", "peerdas_kat.npz"))["srs_monomial_compressed"].tobytes())
        print(json.dumps({"gpu": bench.gpu_identity(0), "reps": a.reps, "verify": verify(ctx, vsizes, a.reps)}), flush=True)
        ctx.delete()
        return
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
    out["verify"] = verify(ctx, vsizes, a.reps)
    out["verify4844"] = verify4844(ctx, v4sizes, a.reps)
    ctx.delete()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
