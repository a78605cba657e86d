#!/usr/bin/env python3
"""POINT_EVALUATION benchmark: the batch entry ctt_b200_eth_evm_kzg_point_evaluation_batch at n valid calls.

Inputs: the true verify_kzg_proof vectors of tests/golden/kzg_verify_kat.npz whose commitment and proof are finite points, plus geth's
vector (tests/golden/evm_kzg_point_evaluation_kat.json), as precompile records with their versioned hashes, repeated to n. A record's
cost does not depend on which valid opening it holds, except that infinity points skip work, so none are used. Per size: the median
over --reps calls after --warmup of the wall time (host clock around the C entry, which ends in a device synchronise; the statuses are
checked outside the timed region) and of the four phases of ctt_b200_eth_kzg_last_point_eval_timing: host packing and statuses, the
record kernel, the Miller loops, the products with the final exponentiations (CUDA events). The card's name and power limit are read
in the same run. For reference only: the per-call time of the host-only ctt_b200_eth_kzg_verify_kzg_proof, on one host thread. Prints a
table and one JSON line; writes nothing.

  python tools/bench_evm_kzg_point_evaluation.py [--reps 10] [--warmup 2] [--sizes 1,64,1024,16384,65536]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def records():
    """(precompile records, (C, z, y, pi) tuples) of the valid openings with finite points"""
    import evm_kzg_point_evaluation_exact as PE
    g = os.path.join(ROOT, "tests", "golden")
    cases = json.loads(str(np.load(os.path.join(g, "kzg_verify_kat.npz"))["cases"]))["verify_kzg_proof"]
    opens = [tuple(bytes.fromhex(c[k]) for k in ("commitment", "z", "y", "proof")) for c in cases if c["outcome"] == 0]
    with open(os.path.join(g, "evm_kzg_point_evaluation_kat.json")) as f:
        geth = bytes.fromhex(json.load(f)["vectors"][0]["input"])
    _, z, y, c, p = PE.split(geth)
    opens.append((c, z, y, p))
    opens = [o for o in opens if not (o[0][0] & 0x40 or o[3][0] & 0x40)]
    return [PE.record(*o) for o in opens], opens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sizes", default="1,64,1024,16384,65536")
    args = ap.parse_args()
    from constantine_b200 import _lib
    from constantine_b200 import msm as M
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    g = os.path.join(ROOT, "tests", "golden")
    ctx = M.EthKzgContext(np.load(os.path.join(g, "kzg_commit_kat.npz"))["srs_lagrange_brp_compressed"].tobytes(), compressed=True)
    ctx.load_g2_setup(np.load(os.path.join(g, "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes())
    recs, opens = records()
    rows = []
    for n in [int(s) for s in args.sizes.split(",")]:
        data = b"".join(recs[i % len(recs)] for i in range(n))
        r = ctypes.create_string_buffer(64 * n)
        st = ctypes.create_string_buffer(n)
        walls, phases = [], []
        for it in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            rc = lib.ctt_b200_eth_evm_kzg_point_evaluation_batch(ctx._h, r, st, data, n)
            wall = (time.perf_counter() - t0) * 1e3
            assert rc == 0 and st.raw == bytes(n)
            if it >= args.warmup:
                walls.append(wall)
                phases.append(ctx.last_point_eval_timing())
        w = statistics.median(walls)
        row = dict(n=n, wall_ms=round(w, 3), calls_per_s=round(n / w * 1e3))
        for k in ("ms_host", "ms_records", "ms_miller", "ms_final"):
            row[k] = round(statistics.median(p[k] for p in phases), 3)
        rows.append(row)
    host = []
    for it in range(1 + 5):
        c, z, y, p = opens[it % len(opens)]
        t0 = time.perf_counter()
        assert ctx.verify_kzg_proof(c, z, y, p)
        if it:
            host.append((time.perf_counter() - t0) * 1e3)
    ctx.delete()
    host_ms = statistics.median(host)
    gpu = card()
    print("card: %s" % gpu)
    print("%7s %10s %10s %10s %10s %10s %12s" % ("n", "wall ms", "host ms", "records ms", "miller ms", "final ms", "calls/s"))
    for x in rows:
        print("%7d %10.3f %10.3f %10.3f %10.3f %10.3f %12d" % (x["n"], x["wall_ms"], x["ms_host"], x["ms_records"], x["ms_miller"],
                                                              x["ms_final"], x["calls_per_s"]))
    print("for reference, the host-only ctt_b200_eth_kzg_verify_kzg_proof on one host thread: %.3f ms per call" % host_ms)
    print(json.dumps({"bench": "evm_kzg_point_evaluation", "card": gpu, "reps": args.reps, "warmup": args.warmup, "rows": rows,
                      "host_verify_kzg_proof_ms_one_thread": round(host_ms, 3)}))


if __name__ == "__main__":
    main()
