#!/usr/bin/env python3
"""ECRECOVER benchmark: the batch entry ctt_b200_eth_evm_ecrecover_batch at 2^16 and 2^20 records.

Inputs: valid signatures from tests/evm_ecrecover_exact.py's bulk builder (16 keys, 16 nonces, random digests; every record
recovers its key, and the kernel's cost does not depend on which valid signature a record holds). Per size: the median over --reps
calls after --warmup of the wall time (host clock around the C entry alone, which ends in a device synchronise; statuses are checked
outside the timed region) and of the kernel time from ctt_b200_eth_evm_ecops_last_timing (CUDA events), and records per second of
each. The card's name and power limit are read in the same run. As a CPU point of reference, when the `cryptography` package is
importable: OpenSSL's ECDSA verify rate on one core over the same digests (the same double-scalar multiplication). Prints a table
and one JSON line; writes nothing.

  python tools/bench_evm_ecrecover.py [--reps 10] [--warmup 2] [--sizes 65536,1048576]
"""
import argparse
import ctypes
import json
import os
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


def openssl_verify_rate(recs, seconds=2.0):
    """verifications per second on one core, or None when `cryptography` is not importable"""
    try:
        from cryptography.hazmat.primitives import hashes
        from cryptography.hazmat.primitives.asymmetric import ec
        from cryptography.hazmat.primitives.asymmetric.utils import Prehashed, encode_dss_signature
    except ImportError:
        return None
    import evm_ecrecover_exact as E
    items = []
    for inp in recs[:256]:
        m, _, r, s = E.parse(inp)
        pub = E.recover_closed(m % E.N, r, s, inp[63] == 27)
        key = ec.EllipticCurvePublicNumbers(pub[0], pub[1], ec.SECP256K1()).public_key()
        items.append((key, encode_dss_signature(r, s), inp[:32]))
    algo = ec.ECDSA(Prehashed(hashes.SHA256()))
    done, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        for key, sig, dg in items:
            key.verify(sig, dg, algo)
        done += len(items)
    return done / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sizes", default="65536,1048576")
    args = ap.parse_args()
    import evm_ecrecover_exact as E
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    recs, _ = E.bulk_records(4096, seed=1)
    block = b"".join(recs)
    rows = []
    for n in sizes:
        data = (block * (n // 4096 + 1))[:n * 128]
        r = ctypes.create_string_buffer(n * 32)
        st = ctypes.create_string_buffer(n)
        walls, kernels = [], []
        for it in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            rc = lib.ctt_b200_eth_evm_ecrecover_batch(r, st, data, n)
            wall = (time.perf_counter() - t0) * 1e3
            assert rc == 0 and st.raw == bytes(n)
            ms = ctypes.c_float(0)
            lib.ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(ms))
            if it >= args.warmup:
                walls.append(wall)
                kernels.append(ms.value)
        w, k = statistics.median(walls), statistics.median(kernels)
        rows.append(dict(n=n, wall_ms=round(w, 3), kernel_ms=round(k, 3), wall_per_s=round(n / w * 1e3), kernel_per_s=round(n / k * 1e3)))
    cpu = openssl_verify_rate(recs)
    gpu = card()
    print("card: %s" % gpu)
    print("%9s %11s %11s %14s %14s" % ("n", "wall ms", "kernel ms", "wall rec/s", "kernel rec/s"))
    for x in rows:
        print("%9d %11.3f %11.3f %14d %14d" % (x["n"], x["wall_ms"], x["kernel_ms"], x["wall_per_s"], x["kernel_per_s"]))
    print("OpenSSL ECDSA verify, one CPU core: %s" % ("%.0f / s" % cpu if cpu else "not measured (cryptography not importable)"))
    print(json.dumps({"bench": "evm_ecrecover", "card": gpu, "reps": args.reps, "warmup": args.warmup, "rows": rows,
                      "openssl_verify_per_s_one_core": round(cpu) if cpu else None}))


if __name__ == "__main__":
    main()
