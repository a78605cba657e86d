#!/usr/bin/env python3
"""EIP-197 ecPairing benchmark on BN254: ctt_b200_eth_evm_bn254_ecpairingcheck_batch at calls x pairs = 1 x 2, 1 x 128, 64 x 4,
1024 x 4 and 16384 x 4.

Every call is true: its pairs are (G1, G2) and (G1, -G2) alternately (the decoder, the subgroup tests, the Miller loops and the final
exponentiations cost the same for any valid points). Per shape: the median wall time of the C entry over --reps calls after --warmup
(host clock around a call that ends in a device synchronise), the device phases of the same calls from
ctt_b200_eth_evm_bn254_last_timing (medians), and checks per second. The card's name and power limit are read in the same run.
Prints a table and one JSON line; writes nothing.

  python tools/bench_bn254_pairing.py [--reps 10] [--warmup 2]
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

SHAPES = [(1, 2), (1, 128), (64, 4), (1024, 4), (16384, 4)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import bn254_exact as B
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    pos, neg = B.encode_pair(B.G1_GEN, B.G2_GEN), B.encode_pair(B.G1_GEN, B.g2_neg(B.G2_GEN))
    rows = []
    for ncalls, npairs in SHAPES:
        call = (pos + neg) * (npairs // 2)
        data = call * ncalls
        offsets = (ctypes.c_size_t * (ncalls + 1))(*[i * len(call) for i in range(ncalls + 1)])
        r = ctypes.create_string_buffer(32 * ncalls)
        st = ctypes.create_string_buffer(ncalls)
        walls, phases = [], []
        for it in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            rc = lib.ctt_b200_eth_evm_bn254_ecpairingcheck_batch(r, st, data, len(data), offsets, ncalls)
            wall = (time.perf_counter() - t0) * 1e3
            assert rc == 0 and st.raw == bytes(ncalls) and all(r.raw[32 * i + 31] == 1 for i in range(ncalls))
            v = [ctypes.c_float(0) for _ in range(4)]
            lib.ctt_b200_eth_evm_bn254_last_timing(*[ctypes.byref(x) for x in v])
            if it >= args.warmup:
                walls.append(wall)
                phases.append([x.value for x in v])
        med = statistics.median(walls)
        ph = [statistics.median(p[k] for p in phases) for k in range(4)]
        rows.append({"calls": ncalls, "pairs_per_call": npairs, "wall_ms": round(med, 3), "host_ms": round(ph[0], 3),
                     "decode_ms": round(ph[1], 3), "miller_ms": round(ph[2], 3), "final_ms": round(ph[3], 3),
                     "checks_per_s": round(ncalls / (med / 1e3), 1)})
    gpu = card()
    print("card: %s" % gpu)
    print("%8s %6s %10s %9s %10s %10s %10s %12s" % ("calls", "pairs", "wall ms", "host ms", "decode ms", "miller ms", "final ms", "checks/s"))
    for x in rows:
        print("%8d %6d %10.3f %9.3f %10.3f %10.3f %10.3f %12.1f" % (x["calls"], x["pairs_per_call"], x["wall_ms"], x["host_ms"],
                                                                   x["decode_ms"], x["miller_ms"], x["final_ms"], x["checks_per_s"]))
    print(json.dumps({"bench": "bn254_ecpairingcheck", "card": gpu, "reps": args.reps, "rows": rows}))


if __name__ == "__main__":
    main()
