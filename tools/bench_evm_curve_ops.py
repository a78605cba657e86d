#!/usr/bin/env python3
"""EVM curve-operation benchmark: the six batch entries ctt_b200_eth_evm_{bn254_g1add, bn254_g1mul, bls12381_g1add, bls12381_g2add,
bls12381_g1mul, bls12381_g2mul}_batch at n = 1, 4096, 65536 and 2^20 records.

Inputs: 1024 distinct valid records tiled to n (points [k]G of random k, random 256-bit scalars; every record succeeds, and the
kernels' cost does not depend on which valid point a record holds). Per shape: the median over --reps calls after --warmup of the
wall time (host clock around the C entry alone, which ends in a device synchronise; statuses are checked outside the timed region)
and of the kernel time from ctt_b200_eth_evm_ecops_last_timing (CUDA events). The card's name and power limit are read in the same
run. Prints a table and one JSON line; writes nothing.

  python tools/bench_evm_curve_ops.py [--reps 10] [--warmup 2] [--sizes 1,4096,65536,1048576]
"""
import argparse
import ctypes
import json
import os
import random
import statistics
import subprocess
import sys
import time

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


def distinct_records(op, rnd, count=1024):
    import eip2537_exact as E
    import evm_curve_ops_exact as X
    if op.startswith("bn254"):
        pts = [X.bn_mul(rnd.randrange(1, X.BN_R), X.BN_G1) for _ in range(16)]
        enc = X.bn_enc
    else:
        g = E.G2 if "g2" in op else E.G1
        pts = [E.ec_mul(rnd.randrange(1, X.BLS_R), E.generator(g)) for _ in range(16)]
        enc = lambda pt: E.enc_point(g, pt)   # noqa: E731
    if op.endswith("mul"):
        return [enc(pts[i % 16]) + rnd.getrandbits(256).to_bytes(32, "big") for i in range(count)]
    return [enc(pts[i % 16]) + enc(pts[(i * 7 + 3) % 16]) for i in range(count)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sizes", default="1,4096,65536,1048576")
    args = ap.parse_args()
    import evm_curve_ops_exact as X
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    rnd = random.Random(196)
    rows = []
    for op in X.OPS:
        n_in, n_out = X.SIZES[op]
        block = b"".join(distinct_records(op, rnd))
        fn = getattr(lib, "ctt_b200_eth_evm_%s_batch" % op)
        for n in sizes:
            data = (block * (n // 1024 + 1))[:n * n_in]
            r = ctypes.create_string_buffer(n * n_out)
            st = ctypes.create_string_buffer(n)
            walls, kernels = [], []
            for it in range(args.warmup + args.reps):
                t0 = time.perf_counter()
                rc = fn(r, st, data, n)
                wall = (time.perf_counter() - t0) * 1e3
                assert rc == 0 and st.raw == bytes(n)
                ms = ctypes.c_float(0)
                lib.ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(ms))
                if it >= args.warmup:
                    walls.append(wall)
                    kernels.append(ms.value)
            rows.append(dict(entry=op, n=n, wall_ms=round(statistics.median(walls), 3),
                             kernel_ms=round(statistics.median(kernels), 3)))
    gpu = card()
    print("card: %s" % gpu)
    print("%-16s %9s %11s %11s" % ("entry", "n", "wall ms", "kernel ms"))
    for x in rows:
        print("%-16s %9d %11.3f %11.3f" % (x["entry"], x["n"], x["wall_ms"], x["kernel_ms"]))
    print(json.dumps({"bench": "evm_curve_ops", "card": gpu, "reps": args.reps, "warmup": args.warmup, "rows": rows}))


if __name__ == "__main__":
    main()
